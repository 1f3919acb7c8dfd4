"""GPU: utils.rgb_lpips (k4_lpips_forward, csrc/k4_lpips.cu) on seeded random weights of the real shapes, against the
float64 restatement of oracle/lpips.py: every VGG16 layer element by element (k4_testing_lpips_stage), the pools and
the head exactly or to an fp64 bound, and the whole score no further from fp64 than torch's own fp32 / TF32 cuDNN
evaluation of the same net, from 64 x 64 to a 4032 x 3024 pair; AlexNet the same way; no host synchronisation,
bitwise repeats, strided views, both render paths and the errors."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from k4nerf import _lib, render, utils
from k4nerf.utils import LpipsNet, rgb_lpips
from helpers import make_state, model_from_state
from oracle import lpips as ol
from oracle import scenes

pytestmark = pytest.mark.gpu

K4_ERR_INVALID_ARG, K4_ERR_WORKSPACE = -1, -4
_NETS = {}


def _net(name, dev, seed=0):
    key = (name, dev, seed)
    if key not in _NETS:
        sd = ol.random_state_dict(name, seed=seed)
        _NETS[key] = (sd, LpipsNet(name, sd, dev))
    return _NETS[key]


def _image(H, W, g):
    """A smooth random image in [0, 1], [H, W, 3] fp32 (CPU)."""
    a = torch.rand(1, 3, H, W, generator=g, dtype=torch.float64)
    a = F.avg_pool2d(a, 5, stride=1, padding=2, count_include_pad=False)[0]
    a = (a - a.mean()) * 3 + 0.5
    return a.clamp(0, 1).permute(1, 2, 0).float().contiguous()


def _pair(H, W, kind, seed):
    g = torch.Generator().manual_seed(seed)
    a = _image(H, W, g)
    if kind == 'same':
        return a, a.clone()
    if kind == 'near':
        return a, (a + 0.01 * torch.randn(H, W, 3, generator=g)).clamp(0, 1)
    return a, _image(H, W, g)


def _chw(x, dev):
    return x.permute(2, 0, 1).to(dev)


def _stage(net, img, s):
    """k4_testing_lpips_stage: (h, w, c) NHWC tensor of stage s of one [H, W, 3] CUDA image."""
    lib = _lib.lib
    H, W = img.shape[0], img.shape[1]
    ws = torch.empty(lib.k4_lpips_workspace_bytes(net.handle, H, W), dtype=torch.uint8, device=img.device)
    shape = (C.c_int64 * 3)()
    stream = C.c_void_p(torch.cuda.current_stream(img.device).cuda_stream)
    args = lambda out: (net.handle, C.c_void_p(img.data_ptr()), utils._strides3(img), H, W, s, out, shape,
                        C.c_void_p(ws.data_ptr()), ws.numel(), stream)
    _lib.check(lib.k4_testing_lpips_stage(*args(None)), 'k4_testing_lpips_stage')
    dt = torch.float16 if net.net_name == 'vgg' else torch.float32
    out = torch.empty(tuple(shape), dtype=dt, device=img.device)
    _lib.check(lib.k4_testing_lpips_stage(*args(C.c_void_p(out.data_ptr()))), 'k4_testing_lpips_stage')
    return out


def _split_value(t):
    """A VGG stage [h, w, 3 C] ([hi | lo | hi]) as fp64 hi + lo [1, C, h, w]; the third copy must equal the first."""
    C3 = t.shape[-1] // 3
    assert torch.equal(t[..., 2 * C3:].view(torch.int16), t[..., :C3].view(torch.int16)), 'the second hi copy differs'
    return (t[..., :C3].double() + t[..., C3:2 * C3].double()).permute(2, 0, 1)[None]


# ------------------------------------------------------------------------------------------------
# per layer
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,W', [(64, 64), (37, 45)])
def test_vgg_layers_against_fp64(cuda_device, H, W):
    """Each stage from the previous GPU stage, every value the fp16 pair hi + lo: the scaled input is the split of
    fp32 (2x - 1 - shift) / scale exactly; a pool equals max_pool2d of its input exactly; a convolution (K = 3 Cin: a_hi
    w_hi + a_lo w_hi + a_hi w_lo, fp32 accumulation, bias + ReLU, output split) is within 2^-16 sum |a||w| of the fp64
    convolution of the input's values with the fp32 weights, plus the dropped a_lo w_lo and weight remainders, a few
    fp32 roundings, and the output split's rounding (2^-22 relative, 2^-25 absolute)."""
    sd, net = _net('vgg', cuda_device)
    a, _ = _pair(H, W, 'far', seed=H * 100 + W)
    img = a.to(cuda_device)
    prev = _stage(net, img, 0)
    v = ol.scale_input(_chw(a, cuda_device), torch.float32)[0].permute(1, 2, 0)
    hi = v.half()
    lo = (v - hi.float()).half()
    assert tuple(prev.shape) == (H, W, 32)
    assert torch.equal(prev[..., :9], torch.cat([hi, lo, hi], -1)) and not bool(prev[..., 9:].any())
    prev = prev[..., :9]
    for i, (kind, p, _) in enumerate(ol.OPS['vgg']):
        got = _stage(net, img, i + 1)
        a64, g64 = _split_value(prev), _split_value(got)
        if kind == 'pool':
            assert torch.equal(g64, F.max_pool2d(a64, 2, 2)), f'stage {i + 1}: pool'
        else:
            k = ol.CONVS['vgg'][p][0]
            w = sd[k + '.weight'].to(cuda_device)
            w_hi = w.half().float()
            w_lo = (w - w_hi).half().float()
            b = sd[k + '.bias'].to(cuda_device).double()
            C = a64.shape[1]
            a_lo = prev[..., C:2 * C].double().permute(2, 0, 1)[None]
            ref = F.relu(F.conv2d(a64, w.double(), b, padding=1))
            S = F.conv2d(a64.abs(), w.double().abs(), padding=1)
            drop = (F.conv2d(a_lo.abs(), w_lo.double().abs(), padding=1) +
                    F.conv2d(a64.abs(), (w.double() - w_hi.double() - w_lo.double()).abs(), padding=1))
            e = 2.0 ** -16 * S + drop + 2.0 ** -22 * (ref.abs() + b.abs().max().item())
            bound = e + 2.0 ** -21 * (ref.abs() + e) + 2.0 ** -24
            err = (g64 - ref).abs()
            assert tuple(g64.shape) == tuple(ref.shape), (i, g64.shape, ref.shape)
            assert bool((err <= bound).all()), f'stage {i + 1} ({k}): worst excess {(err - bound).max().item():.3e}'
            assert bool((g64 > 0).any()), f'stage {i + 1}: all zero, the case lost its point'
        prev = got


@pytest.mark.parametrize('H,W', [(67, 75), (131, 257)])
def test_alex_layers_against_fp64(cuda_device, H, W):
    """fp32 direct convolutions within n 2^-24 sum |a||w| of fp64 (n the products per output); pools exact."""
    sd, net = _net('alex', cuda_device)
    a, _ = _pair(H, W, 'far', seed=H * 100 + W + 1)
    img = a.to(cuda_device)
    prev = _stage(net, img, 0)
    assert torch.equal(prev, ol.scale_input(_chw(a, cuda_device), torch.float32)[0].permute(1, 2, 0))
    for i, (kind, p, b) in enumerate(ol.OPS['alex']):
        got = _stage(net, img, i + 1).double()
        a64 = prev.double().permute(2, 0, 1)[None]
        if kind == 'pool':
            assert torch.equal(got, F.max_pool2d(a64, p, b)[0].permute(1, 2, 0)), f'stage {i + 1}: pool'
        else:
            k, ci, _, ks, s, pad = ol.CONVS['alex'][p]
            w = sd[k + '.weight'].to(cuda_device).double()
            ref = F.relu(F.conv2d(a64, w, sd[k + '.bias'].to(cuda_device).double(), stride=s, padding=pad))[0].permute(1, 2, 0)
            S = F.conv2d(a64.abs(), w.abs(), stride=s, padding=pad)[0].permute(1, 2, 0)
            bound = (ci * ks * ks + 2) * 2.0 ** -24 * (S + sd[k + '.bias'].abs().max().item())
            assert tuple(got.shape) == tuple(ref.shape)
            assert bool(((got - ref).abs() <= bound).all()), f'stage {i + 1} ({k})'
        prev = got.float()


def test_head_is_fp64_of_the_gpu_taps(cuda_device):
    """The score equals the fp64 head of the GPU's own taps (VGG: the values hi + lo) to 1e-12 relative: the head and
    the reduction add nothing beyond fp64 rounding."""
    for name, (H, W) in (('vgg', (45, 70)), ('alex', (75, 91))):
        sd, net = _net(name, cuda_device)
        a, b = _pair(H, W, 'near', seed=11)
        i0, i1 = a.to(cuda_device), b.to(cuda_device)
        taps = [(s + 1) for s, (kind, _, t) in enumerate(ol.OPS[name]) if kind == 'conv' and t is not None]
        ref = 0.0
        for k, s in enumerate(taps):
            f0, f1 = _stage(net, i0, s), _stage(net, i1, s)
            if name == 'vgg':
                f0, f1 = _split_value(f0), _split_value(f1)
            else:
                f0, f1 = f0.double().permute(2, 0, 1)[None], f1.double().permute(2, 0, 1)[None]
            ref = ref + ol.head(sd, k, f0, f1).item()
        got = net(i0, i1)
        assert abs(got - ref) <= 1e-12 * ref, (name, got, ref)


# ------------------------------------------------------------------------------------------------
# whole score
# ------------------------------------------------------------------------------------------------
def _criterion(name, sd, net, a, b, dev):
    """|GPU - fp64| <= |torch fp32 (cuDNN, default TF32) - fp64|; returns the three values."""
    a_d, b_d = a.to(dev), b.to(dev)
    got = net(a_d, b_d)
    with torch.no_grad():
        ref = ol.lpips(sd, name, _chw(a, dev), _chw(b, dev), torch.float64).item()
        t32 = ol.lpips(sd, name, _chw(a, dev), _chw(b, dev), torch.float32).item()
    torch.cuda.empty_cache()
    assert abs(got - ref) <= abs(t32 - ref), (name, got, ref, t32)
    return got, ref, t32


@pytest.mark.parametrize('kind', ['same', 'near', 'far'])
@pytest.mark.parametrize('H,W', [(64, 64), (131, 257), (756, 1008)])
def test_vgg_score_meets_the_torch_tf32_criterion(cuda_device, H, W, kind):
    sd, net = _net('vgg', cuda_device)
    a, b = _pair(H, W, kind, seed=H + W)
    got, ref, _ = _criterion('vgg', sd, net, a, b, cuda_device)
    if kind == 'same':
        assert got == 0.0
    else:
        assert ref > 0 and got > 0


def test_vgg_score_of_a_4k_pair(cuda_device):
    sd, net = _net('vgg', cuda_device)
    a, b = _pair(3024, 4032, 'near', seed=4)
    _criterion('vgg', sd, net, a, b, cuda_device)


@pytest.mark.parametrize('kind', ['same', 'near', 'far'])
@pytest.mark.parametrize('H,W', [(64, 64), (131, 257), (756, 1008)])
def test_alex_score_meets_the_torch_tf32_criterion(cuda_device, H, W, kind):
    sd, net = _net('alex', cuda_device)
    a, b = _pair(H, W, kind, seed=H + W + 7)
    got, ref, _ = _criterion('alex', sd, net, a, b, cuda_device)
    if kind == 'same':
        assert got == 0.0


# ------------------------------------------------------------------------------------------------
# the call itself
# ------------------------------------------------------------------------------------------------
def test_forward_does_not_synchronise_and_repeats_bitwise(cuda_device):
    sd, net = _net('vgg', cuda_device)
    a, b = _pair(756, 1008, 'far', seed=9)
    a, b = a.to(cuda_device), b.to(cuda_device)
    lib = _lib.lib
    ws = torch.empty(lib.k4_lpips_workspace_bytes(net.handle, 756, 1008), dtype=torch.uint8, device=cuda_device)
    out = torch.empty(3, dtype=torch.float64, device=cuda_device)
    stream = C.c_void_p(torch.cuda.current_stream(cuda_device).cuda_stream)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for i in range(3):
            _lib.check(lib.k4_lpips_forward(net.handle, C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), utils._strides3(a),
                                            utils._strides3(b), 756, 1008, C.c_void_p(out.data_ptr() + 8 * i),
                                            C.c_void_p(ws.data_ptr()), ws.numel(), stream))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    v = out.cpu()
    assert v[0].item() > 0 and torch.equal(v[0].view(torch.int64), v[1].view(torch.int64))
    assert torch.equal(v[0].view(torch.int64), v[2].view(torch.int64))
    assert rgb_lpips(a, b, 'vgg', weights=sd) == v[0].item()


def test_inputs_are_read_in_place_through_strides(cuda_device):
    """A [3, H, W] frame as permute(1, 2, 0), a crop and numpy arrays give the contiguous pair's score bit for bit."""
    sd, net = _net('vgg', cuda_device)
    a, b = _pair(70, 90, 'far', seed=12)
    want = net(a.to(cuda_device), b.to(cuda_device))
    chw = b.permute(2, 0, 1).contiguous().to(cuda_device)
    assert net(a.to(cuda_device), chw.permute(1, 2, 0)) == want
    big = torch.zeros(80, 100, 3)
    big[5:75, 7:97] = a
    assert net(big.to(cuda_device)[5:75, 7:97], b.to(cuda_device)) == want
    assert rgb_lpips(a.numpy(), b.numpy(), 'vgg', device=cuda_device, weights=sd) == want
    assert rgb_lpips(a.double().to(cuda_device), b.to(cuda_device), 'vgg', weights=sd) == want


def test_errors(cuda_device):
    sd, net = _net('vgg', cuda_device)
    lib = _lib.lib
    assert lib.k4_lpips_workspace_bytes(net.handle, 15, 64) == 0
    assert lib.k4_lpips_workspace_bytes(net.handle, 16, 16) > 0
    assert lib.k4_lpips_workspace_bytes(_net('alex', cuda_device)[1].handle, 30, 64) == 0
    assert lib.k4_lpips_workspace_bytes(_net('alex', cuda_device)[1].handle, 31, 31) > 0
    assert lib.k4_lpips_workspace_bytes(net.handle, 64, 16385) == 0
    with pytest.raises(ValueError):
        rgb_lpips(torch.rand(15, 40, 3, device=cuda_device), torch.rand(15, 40, 3, device=cuda_device), 'vgg', weights=sd)
    with pytest.raises(ValueError):
        rgb_lpips(torch.rand(20, 40, 3, device=cuda_device), torch.rand(20, 41, 3, device=cuda_device), 'vgg', weights=sd)
    with pytest.raises(ValueError):
        rgb_lpips(torch.rand(20, 40, 3), torch.rand(20, 40, 3), 'vgg', device='cpu', weights=sd)
    with pytest.raises(ValueError):
        rgb_lpips(torch.rand(20, 40, 3), torch.rand(20, 40, 3), 'squeeze', device=cuda_device, weights=sd)
    bad = dict(sd)
    bad['scaling_layer.scale'] = torch.ones(1, 3, 1, 1)
    with pytest.raises(ValueError):
        LpipsNet('vgg', bad, cuda_device)
    bad = dict(sd)
    del bad['lin3.model.1.weight']
    with pytest.raises(KeyError):
        LpipsNet('vgg', bad, cuda_device)
    a = torch.rand(32, 32, 3, device=cuda_device)
    st = utils._strides3(a)
    n = lib.k4_lpips_workspace_bytes(net.handle, 32, 32)
    ws = torch.empty(n + 256, dtype=torch.uint8, device=cuda_device)
    out = torch.empty(1, dtype=torch.float64, device=cuda_device)
    call = lambda H=32, W=32, w=ws.data_ptr(), nb=n, o=out.data_ptr(): lib.k4_lpips_forward(
        net.handle, C.c_void_p(a.data_ptr()), C.c_void_p(a.data_ptr()), st, st, H, W, C.c_void_p(o), C.c_void_p(w), nb, None)
    assert call(H=15) == K4_ERR_INVALID_ARG
    assert call(w=ws.data_ptr() + 128) == K4_ERR_INVALID_ARG
    assert call(o=out.data_ptr() + 4) == K4_ERR_INVALID_ARG
    assert call(nb=n - 1) == K4_ERR_WORKSPACE
    assert call() == 0
    torch.cuda.synchronize()
    assert out.item() == 0.0


# ------------------------------------------------------------------------------------------------
# render paths and the lpips package
# ------------------------------------------------------------------------------------------------
def _scene(dev):
    m = model_from_state(make_state('cfgA', res=32, regime='fog'), dev)
    m.mlp_mode = 'fp32'
    H, W = 40, 48
    poses, Ks = [], []
    for th in (30.0, 120.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    rng = np.random.default_rng(5)
    gt = [np.clip(0.5 + 0.3 * rng.standard_normal((H, W, 3)), 0, 1).astype(np.float32) for _ in range(2)]
    return m, np.array(poses), np.array([[H, W]] * 2), np.array(Ks), gt


def test_render_viewpoints_scores_lpips(cuda_device, monkeypatch, capsys):
    """eval_lpips_vgg / eval_lpips_alex: the returned list is rgb_lpips of each returned frame, both means are printed,
    and the arrays are those of a run without them; render_viewpoints_sr prints the same means."""
    sds = {n: ol.random_state_dict(n, seed=21) for n in ('vgg', 'alex')}
    monkeypatch.setattr(utils, '_lpips_state_dict', lambda name: sds[name])
    monkeypatch.setattr(utils, '__LPIPS__', {})
    m, poses, HW, Ks, gt = _scene(cuda_device)
    kw = dict(scenes.RENDER_KW_DVGO)
    capsys.readouterr()
    on = render.render_viewpoints(m, poses, HW, Ks, False, kw, gt_imgs=gt, eval_lpips_vgg=True, eval_lpips_alex=True)
    out = capsys.readouterr().out.splitlines()
    off = render.render_viewpoints(m, poses, HW, Ks, False, kw, gt_imgs=gt)
    for x, y in zip(on[:4], off[:4]):
        assert np.array_equal(np.asarray(x), np.asarray(y))
    want_vgg = [rgb_lpips(on[0][i], gt[i], 'vgg', device=cuda_device, weights=sds['vgg']) for i in range(2)]
    want_alex = [rgb_lpips(on[0][i], gt[i], 'alex', device=cuda_device, weights=sds['alex']) for i in range(2)]
    assert on[5] == want_vgg and all(v > 0 for v in want_vgg)
    printed = {l.split('(')[1].split(')')[0]: float(l.split()[3]) for l in out if l.startswith('Testing lpips')}
    assert printed == {'vgg': pytest.approx(np.mean(want_vgg), rel=1e-12), 'alex': pytest.approx(np.mean(want_alex), rel=1e-12)}
    render.render_viewpoints_sr(m, poses, HW, Ks, False, kw, gt_imgs=gt, eval_lpips_vgg=True, eval_lpips_alex=True)
    out = capsys.readouterr().out.splitlines()
    printed = {l.split('(')[1].split(')')[0]: float(l.split()[3]) for l in out if l.startswith('Testing lpips')}
    assert printed == {'vgg': pytest.approx(np.mean(want_vgg), rel=1e-12), 'alex': pytest.approx(np.mean(want_alex), rel=1e-12)}


def test_without_the_lpips_package_the_default_weights_raise_import_error(cuda_device, monkeypatch):
    try:
        import lpips  # noqa: F401
        pytest.skip('the lpips package is installed: its weights load')
    except ImportError:
        pass
    monkeypatch.setattr(utils, '__LPIPS__', {})
    with pytest.raises(ImportError):
        rgb_lpips(np.zeros((32, 32, 3), np.float32), np.zeros((32, 32, 3), np.float32), 'vgg', device=cuda_device)


@pytest.mark.parametrize('name', ['vgg', 'alex'])
def test_matches_the_lpips_package(cuda_device, name):
    try:
        import lpips
    except ImportError:
        pytest.skip('the lpips package is not installed: nothing to compare lpips.LPIPS with (the fp64 restatement in '
                    'oracle/lpips.py stands in for it above)')
    model = lpips.LPIPS(net=name, version='0.1', pretrained=False, pnet_rand=True, verbose=False).eval()
    sd = ol.random_state_dict(name, seed=31)
    model.load_state_dict({k: sd.get(k, v) if not k.startswith('lins.') else sd[k.replace('lins.', 'lin', 1)]
                           for k, v in model.state_dict().items()})
    model = model.to(cuda_device)
    a, b = _pair(131, 257, 'far', seed=32)
    with torch.no_grad():
        pkg = model(_chw(a, cuda_device), _chw(b, cuda_device), normalize=True).item()
        ref = ol.lpips(sd, name, _chw(a, cuda_device), _chw(b, cuda_device)).item()
    got = rgb_lpips(a.to(cuda_device), b.to(cuda_device), name, weights=sd)
    assert abs(got - ref) <= abs(pkg - ref), (got, ref, pkg)
