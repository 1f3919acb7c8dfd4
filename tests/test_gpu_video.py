"""GPU: the video streams of run_sr.py --render_video on the device (csrc/k4_video.cu) bit for bit against the numpy
path -- utils.depth_video_frames' masked percentiles and rainbow frames from one value to 120 LR frames, ties, views,
edge values and every flip / rotation; and render.render_video_4k against render_frame_4k, render_viewpoints_sr and
the reference-structured host path (render_viewpoints_sr, tile_process, numpy) for x1 / x4 decoders and num_cond 1 /
63 / 64."""
import numpy as np
import pytest
import torch

import k4nerf
from k4nerf import render
from k4nerf.sr_esrnet import sft_condition
from k4nerf.utils import depth_video_frames, to8b
from helpers import make_state, model_from_state
from oracle import scenes, sftnet
from test_sftnet_x1 import x1_state_dict
from test_video import _literal

pytestmark = pytest.mark.gpu


def _depths(n, H, W, seed, sel=0.6, levels=None):
    g = torch.Generator().manual_seed(seed)
    d = 2 + torch.randn(n, H, W, 1, generator=g)
    if levels:
        d = torch.round(d * levels) / levels                     # few distinct values: long tie runs
    bg = torch.rand(n, H, W, 1, generator=g) * (0.1 / sel)       # about a fraction `sel` below 0.1
    return d.float(), bg.float().clamp(0, 1)


def _check(depths, bgmaps, dev, **kw):
    """CUDA vs numpy: frames and range bit for bit; returns the range."""
    want, rng_want = depth_video_frames(depths.numpy(), bgmaps.numpy(), return_range=True, **kw)
    got, rng_got = depth_video_frames(depths.to(dev), bgmaps.to(dev), return_range=True, **kw)
    assert got.is_cuda and got.dtype == torch.uint8 and got.is_contiguous()
    assert all(isinstance(v, np.float64) for v in rng_got)
    assert [np.float64(v).tobytes() for v in rng_got] == [np.float64(v).tobytes() for v in rng_want], (rng_got, rng_want)
    assert np.array_equal(got.cpu().numpy(), want)
    return rng_got


@pytest.mark.parametrize('n,H,W', [(1, 1, 1), (1, 1, 2), (1, 3, 1), (2, 7, 5), (3, 64, 257), (4, 300, 401)])
def test_quantiles_and_frames_match_numpy(cuda_device, n, H, W):
    d, b = _depths(n, H, W, seed=n * 1000 + H + W, sel=1.0 if n * H * W < 4 else 0.6)
    dmin, dmax = _check(d, b, cuda_device)
    sel = (d * (1 - b) + b).numpy()[b.numpy() < 0.1]
    want = np.percentile(sel, q=[5, 95])
    assert dmin == want[0] and dmax == want[1]


def test_120_lr_frames(cuda_device):
    """The 120-frame 1008 x 756 depth video: 91 M candidate values."""
    d, b = _depths(120, 756, 1008, seed=7, sel=0.7)
    _check(d, b, cuda_device)


@pytest.mark.parametrize('levels', [1, 4, 1024])
def test_quantised_depths_with_long_ties(cuda_device, levels):
    d, b = _depths(6, 200, 300, seed=levels, levels=levels)
    _check(d, b, cuda_device)


def test_one_all_and_no_selected_values(cuda_device):
    dev = cuda_device
    d, b = _depths(2, 30, 40, seed=3)
    one = torch.full_like(b, 0.5)
    one[1, 17, 9, 0] = 0.05
    assert _check(d, one, dev)[0] == np.float64((d[1, 17, 9, 0] * (1 - one[1, 17, 9, 0]) + one[1, 17, 9, 0]).item())
    _check(d, torch.zeros_like(b), dev)
    with pytest.raises(ValueError):
        depth_video_frames(d.to(dev), torch.full_like(b, 0.1).to(dev))        # bg == 0.1 is not below 0.1


def test_edge_values(cuda_device):
    """dmax == dmin with pixels below, on and above it (colours 255, bad, 0); pixels on dmin and dmax; bg exactly 0.1;
    a NaN depth outside and inside the selection."""
    dev = cuda_device
    d = torch.full((2, 5, 6, 1), 1.5)
    b = torch.zeros(2, 5, 6, 1)
    b[0, 0, :3, 0] = torch.tensor([0.5, 0.6, 1.0])
    d[1, 1, :2, 0] = torch.tensor([9.0, 1.5])
    b[1, 1, :2, 0] = 0.2
    b[1, 2, 2, 0] = 0.1
    assert _check(d, b, dev) == (1.5, 1.5)
    # 21 selected values: (n - 1) q is 1 and 19, so dmin and dmax are values of the frame (colours 255 and 0 there)
    d, b = _depths(1, 3, 7, seed=11, sel=1.0)
    dmin, dmax = _check(d, b, dev)
    dv = (d * (1 - b) + b).double()
    assert bool((dv == dmin).any()) and bool((dv == dmax).any())
    got = depth_video_frames(d.to(dev), b.to(dev)).cpu()
    lut = torch.from_numpy(k4nerf.utils.rainbow_lut_u8())
    assert torch.equal(got[(dv == dmin)[..., 0]], lut[255].expand(1, 3))
    assert torch.equal(got[(dv == dmax)[..., 0]], lut[0].expand(1, 3))
    d, b = _depths(3, 40, 50, seed=11)
    b[0, :4, :4] = 0.1
    d[2, 3, 3, 0] = float('nan')
    b[2, 3, 3, 0] = 0.5
    _check(d, b, dev)
    d[2, 3, 3, 0], b[2, 3, 3, 0] = float('nan'), 0.0
    dmin, dmax = _check(d, b, dev)
    assert np.isnan(dmin) and np.isnan(dmax)


def test_views_are_read_in_place(cuda_device):
    """[n, H, W, 1], [n, H, W], a channel of [n, H, W, 2] and transposed frames give the contiguous results."""
    dev = cuda_device
    d, b = _depths(3, 33, 47, seed=5)
    want, rng = depth_video_frames(d.numpy(), b.numpy(), return_range=True)
    dd, bb = torch.cat([d, -d], -1).to(dev), torch.cat([b, 1 - b], -1).to(dev)
    for x, y in ((d.to(dev), b.to(dev)), (d[..., 0].to(dev), b[..., 0].to(dev)), (dd[..., :1], bb[..., :1]),
                 (dd[..., 0], bb[..., 0])):
        got, r = depth_video_frames(x, y, return_range=True)
        assert np.array_equal(got.cpu().numpy(), want) and r == rng
    dt = d[..., 0].transpose(1, 2).contiguous().to(dev).transpose(1, 2)
    bt = b[..., 0].transpose(1, 2).contiguous().to(dev).transpose(1, 2)
    assert not dt.is_contiguous()
    assert np.array_equal(depth_video_frames(dt, bt).cpu().numpy(), want)


def test_repeated_calls_are_identical(cuda_device):
    d, b = _depths(8, 128, 160, seed=9)
    d, b = d.cuda(cuda_device), b.cuda(cuda_device)
    first = depth_video_frames(d, b, return_range=True)
    for _ in range(3):
        again = depth_video_frames(d, b, return_range=True)
        assert torch.equal(again[0], first[0]) and again[1] == first[1]


@pytest.mark.parametrize('flipy', [False, True])
@pytest.mark.parametrize('rot90', [-1, 0, 1, 2, 3, 4])
def test_depth_frames_flip_and_rotate(cuda_device, flipy, rot90):
    d, b = _depths(2, 19, 31, seed=13)
    _check(d, b, cuda_device, render_video_flipy=flipy, render_video_rot90=rot90)
    want, _ = _literal(d.numpy(), b.numpy(), flipy, rot90)
    got = depth_video_frames(d.to(cuda_device), b.to(cuda_device), render_video_flipy=flipy, render_video_rot90=rot90)
    assert np.array_equal(got.cpu().numpy(), want)


def test_errors(cuda_device):
    dev = cuda_device
    d, b = _depths(2, 8, 9, seed=1)
    with pytest.raises(RuntimeError):
        depth_video_frames(d.to(dev), b)
    with pytest.raises(TypeError):
        depth_video_frames(d.double().to(dev), b.to(dev))
    with pytest.raises(ValueError):
        depth_video_frames(d.to(dev), b[:, 1:].to(dev))
    with pytest.raises(ValueError):
        depth_video_frames(d.to(dev), b.to(dev), q=(5, 101))
    with pytest.raises(ValueError):
        k4nerf.utils.frame_u8_cuda(d.to(dev))


# ------------------------------------------------------------------------------------------------
# render_video_4k
# ------------------------------------------------------------------------------------------------
H, W, N = 20, 28, 3


@pytest.fixture(scope='module')
def scene(cuda_device):
    # the shell regime's surface leaves bgmap < 0.1 on about 16 % of the pixels, which the depth video needs
    m = model_from_state(make_state('cfgA', res=32, regime='shell'), cuda_device)
    m.mlp_mode = 'fp32'                                # sequential per-ray accumulation: frames reproduce bit for bit
    poses, Ks = [], []
    for th in (30.0, 75.0, 120.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    return m, np.array(poses), np.array([[H, W]] * N), np.array(Ks), dict(scenes.RENDER_KW_DVGO)


def _net(dev, scale, nc):
    net = k4nerf.SFTNet(3, scale, 64, 5, 32, nc)
    net.load_state_dict(x1_state_dict(seed=3) if scale == 1 else sftnet.random_state_dict(seed=3, num_cond=nc))
    return net.to(dev)


@pytest.fixture(scope='module', params=[(4, 1), (4, 63), (4, 64), (1, 1)], ids=['x4c1', 'x4c63', 'x4c64', 'x1c1'])
def net(request, cuda_device):
    return _net(cuda_device, *request.param)


def test_sr_frames_are_render_frame_4k(scene, net):
    m, poses, HW, Ks, kw = scene
    s = net.scale
    sr, lr, depth = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16)
    assert sr.shape == (N, s * H, s * W, 3) and lr.shape == depth.shape == (N, H, W, 3)
    assert sr.dtype == lr.dtype == depth.dtype == np.uint8
    for i in range(N):
        u8, _ = render.render_frame_4k(m, net, H, W, Ks[i], poses[i], False, kw, test_tile=16, out_u8=True)
        assert np.array_equal(sr[i], u8.cpu().numpy()), i


def test_streams_are_the_reference_structured_host_path(scene, cuda_device):
    """render_viewpoints_sr, then tile_process per frame, then run_sr.py:1455-1463 in numpy: all three arrays equal."""
    m, poses, HW, Ks, kw = scene
    dev = cuda_device
    net = _net(dev, 4, 1)
    rgbs, depths, bgmaps, _, _, rgb_features = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw)
    rgbsr = []
    for idx, rgbsave in enumerate(rgb_features):
        rgbtest = torch.from_numpy(rgbsave).movedim(-1, 0).unsqueeze(0).to(dev)
        input_cond = torch.from_numpy(depths).movedim(-1, 1)[idx, :, :, :].to(dev)
        rgb_srtest = net.tile_process(rgbtest, input_cond, tile_size=16).to('cpu')
        rgbsr.append(rgb_srtest.squeeze().movedim(0, -1).detach().clamp(0, 1).numpy())
    want_depth, _ = _literal(depths, bgmaps, False, 0)
    sr, lr, depth = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16)
    assert np.array_equal(sr, to8b(np.array(rgbsr)))
    assert np.array_equal(lr, to8b(rgbs))
    assert np.array_equal(depth, want_depth)


@pytest.mark.parametrize('flipy', [False, True])
@pytest.mark.parametrize('rot90', [-1, 0, 1, 2, 3, 4])
def test_flip_and_rotation(scene, cuda_device, flipy, rot90):
    """Every stream is the flipped / rotated default stream; the LR one is to8b of render_viewpoints_sr's rgbs with
    the same flip / rotation."""
    m, poses, HW, Ks, kw = scene
    net = _net(cuda_device, 4, 1)
    base = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16)
    got = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16, render_video_flipy=flipy,
                                 render_video_rot90=rot90)
    for g, b in zip(got, base):
        b = np.flip(b, axis=1) if flipy else b
        assert np.array_equal(g, np.rot90(b, k=rot90, axes=(1, 2)))
    rgbs = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw, render_video_flipy=flipy, render_video_rot90=rot90)[0]
    assert np.array_equal(got[1], to8b(rgbs))


def test_render_factor(scene, cuda_device):
    m, poses, HW, Ks, kw = scene
    net = _net(cuda_device, 4, 1)
    sr, lr, depth = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16, render_factor=2)
    assert sr.shape == (N, 4 * (H // 2), 4 * (W // 2), 3) and lr.shape == depth.shape == (N, H // 2, W // 2, 3)
    rgbs, depths, bgmaps = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw, render_factor=2)[:3]
    assert np.array_equal(lr, to8b(rgbs))
    assert np.array_equal(depth, _literal(depths, bgmaps, False, 0)[0])
    K2 = np.copy(Ks)
    K2[:, :2, :3] /= 2
    u8, _ = render.render_frame_4k(m, net, H // 2, W // 2, K2[1], poses[1], False, kw, test_tile=16, out_u8=True)
    assert np.array_equal(sr[1], u8.cpu().numpy())


def test_on_frame_receives_the_frames(scene, cuda_device):
    m, poses, HW, Ks, kw = scene
    net = _net(cuda_device, 4, 63)
    want = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16, render_video_rot90=1)
    seen = []

    def on_frame(i, sr_u8, lr_u8):
        assert sr_u8.is_cuda and lr_u8.is_cuda and sr_u8.dtype == lr_u8.dtype == torch.uint8
        seen.append((i, sr_u8.cpu().numpy(), lr_u8.cpu().numpy()))
    sr, lr, depth = render.render_video_4k(m, net, poses, HW, Ks, False, kw, test_tile=16, render_video_rot90=1,
                                           on_frame=on_frame)
    assert sr is None and [s[0] for s in seen] == list(range(N))
    assert np.array_equal(np.stack([s[1] for s in seen]), want[0])
    assert np.array_equal(np.stack([s[2] for s in seen]), want[1])
    assert np.array_equal(lr, want[1]) and np.array_equal(depth, want[2])


def test_condition_is_sft_condition_of_the_unflipped_frame(scene, cuda_device):
    """With a flip the decoder still reads the unflipped frame and its own condition (num_cond 64: depth + view)."""
    m, poses, HW, Ks, kw = scene
    dev = cuda_device
    net = _net(dev, 4, 64)
    sr = render.render_video_4k(m, net, poses[:1], HW[:1], Ks[:1], False, kw, test_tile=16, render_video_flipy=True)[0]
    _, depths, _, _, viewdirs, feats = render.render_viewpoints_sr(m, poses[:1], HW[:1], Ks[:1], False, kw)
    x = torch.from_numpy(feats[0]).movedim(-1, 0).unsqueeze(0).to(dev)
    cond = sft_condition(64, torch.from_numpy(depths[0]).to(dev), viewdirs[0], H, W)
    ref = net.tile_process(x, cond, tile_size=16, to_cpu=False).squeeze(0).clamp(0, 1)
    ref8 = (ref * 255).to(torch.uint8).permute(1, 2, 0).cpu().numpy()
    assert np.array_equal(sr[0], np.flip(ref8, axis=0))
