"""CPU: the LPIPS restatement of oracle/lpips.py (the definition the GPU path is held to) without a GPU -- its keys and
shapes, a literal layer-by-layer torch forward in the shape of lpips' own modules, the unbatched broadcast, floor
pooling at odd sizes -- and the argument checks of the C entry points k4_lpips_*."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from oracle import lpips as ol

K4_ERR_INVALID_ARG = -1


def test_keys_and_shapes():
    """The parameters in the C ABI's order, with the shapes of lpips.LPIPS(net=..., version='0.1').state_dict()."""
    vgg = ol.param_keys('vgg')
    assert len(vgg) == 31 and vgg[:4] == ['net.slice1.0.weight', 'net.slice1.0.bias', 'net.slice1.2.weight', 'net.slice1.2.bias']
    assert [k[:-len('.weight')] for k in vgg[0:26:2]] == [
        'net.slice1.0', 'net.slice1.2', 'net.slice2.5', 'net.slice2.7', 'net.slice3.10', 'net.slice3.12', 'net.slice3.14',
        'net.slice4.17', 'net.slice4.19', 'net.slice4.21', 'net.slice5.24', 'net.slice5.26', 'net.slice5.28']
    assert vgg[26:] == [f'lin{i}.model.1.weight' for i in range(5)]
    alex = ol.param_keys('alex')
    assert len(alex) == 15
    assert [k[:-len('.weight')] for k in alex[0:10:2]] == ['net.slice1.0', 'net.slice2.3', 'net.slice3.6', 'net.slice4.8', 'net.slice5.10']
    s = ol.param_shapes('vgg')
    assert s['net.slice1.0.weight'] == (64, 3, 3, 3) and s['net.slice5.28.weight'] == (512, 512, 3, 3)
    assert s['net.slice2.5.bias'] == (128,) and s['lin4.model.1.weight'] == (1, 512, 1, 1)
    s = ol.param_shapes('alex')
    assert s['net.slice1.0.weight'] == (64, 3, 11, 11) and s['net.slice2.3.weight'] == (192, 64, 5, 5)
    assert s['net.slice3.6.weight'] == (384, 192, 3, 3) and s['lin2.model.1.weight'] == (1, 384, 1, 1)
    for net in ('vgg', 'alex'):
        sd = ol.random_state_dict(net, seed=1)
        assert all(tuple(sd[k].shape) == v for k, v in ol.param_shapes(net).items())
        assert tuple(sd['scaling_layer.shift'].shape) == (1, 3, 1, 1)
        assert [sd[f'lin{i}.model.1.weight'].shape[1] for i in range(5)] == list(ol.TAP_CHANNELS[net])


class _ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer('shift', torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer('scale', torch.Tensor([.458, .448, .450])[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale


def _features(net):
    """torchvision's vgg16().features[:30] / alexnet().features[:12], written out, and lpips' slice boundaries."""
    if net == 'vgg':
        cfg = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512]
        layers, c = [], 3
        for v in cfg:
            if v == 'M':
                layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
            else:
                layers += [nn.Conv2d(c, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
                c = v
        return nn.Sequential(*layers), (4, 9, 16, 23, 30)
    layers = [nn.Conv2d(3, 64, kernel_size=11, stride=4, padding=2), nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2),
              nn.Conv2d(64, 192, kernel_size=5, padding=2), nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2),
              nn.Conv2d(192, 384, kernel_size=3, padding=1), nn.ReLU(inplace=True),
              nn.Conv2d(384, 256, kernel_size=3, padding=1), nn.ReLU(inplace=True),
              nn.Conv2d(256, 256, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
    return nn.Sequential(*layers), (2, 5, 8, 10, 12)


def _literal_lpips(sd, net, in0, in1):
    """lpips.LPIPS.forward(in0, in1, normalize=True) with version 0.1, fp32, module by module."""
    feats, bounds = _features(net)
    for k in sd:
        if k.startswith('net.slice'):
            idx, what = int(k.split('.')[2]), k.split('.')[3]
            getattr(feats[idx], what).data.copy_(sd[k])
    scaling = _ScalingLayer()
    lins = []
    for i, c in enumerate(ol.TAP_CHANNELS[net]):
        lin = nn.Sequential(nn.Dropout(), nn.Conv2d(c, 1, 1, stride=1, padding=0, bias=False))
        lin[1].weight.data.copy_(sd[f'lin{i}.model.1.weight'])
        lins.append(lin.eval())

    def taps(x):
        out, lo = [], 0
        for hi in bounds:
            for i in range(lo, hi):
                x = feats[i](x)
            out.append(x)
            lo = hi
        return out

    in0, in1 = 2 * in0 - 1, 2 * in1 - 1
    o0, o1 = taps(scaling(in0)), taps(scaling(in1))
    val = 0
    for k in range(5):
        n0 = o0[k] / (torch.sqrt(torch.sum(o0[k] ** 2, dim=1, keepdim=True)) + 1e-10)
        n1 = o1[k] / (torch.sqrt(torch.sum(o1[k] ** 2, dim=1, keepdim=True)) + 1e-10)
        val = val + lins[k]((n0 - n1) ** 2).mean([2, 3], keepdim=True)
    return val


@pytest.mark.parametrize('net', ['vgg', 'alex'])
def test_literal_forward_equals_the_restatement(net):
    sd = ol.random_state_dict(net, seed=2)
    g = torch.Generator().manual_seed(3)
    H, W = (36, 44) if net == 'vgg' else (67, 75)
    a = torch.rand(3, H, W, generator=g)
    b = (a + 0.2 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    with torch.no_grad():
        lit = _literal_lpips(sd, net, a, b)
        ref = ol.lpips(sd, net, a, b)
        ref32 = ol.lpips(sd, net, a, b, dtype=torch.float32)
    assert lit.shape == ref.shape == (1, 1, 1, 1)
    assert ref.item() > 0
    assert abs(lit.item() - ref.item()) <= 1e-4 * ref.item(), (lit.item(), ref.item())
    assert abs(ref32.item() - ref.item()) <= 1e-4 * ref.item()


def test_unbatched_input_broadcasts_to_a_batch_of_one():
    sd = ol.random_state_dict('vgg', seed=4)
    g = torch.Generator().manual_seed(5)
    a, b = torch.rand(3, 32, 40, generator=g), torch.rand(3, 32, 40, generator=g)
    assert tuple(ol.scale_input(a).shape) == (1, 3, 32, 40)
    with torch.no_grad():
        u = ol.lpips(sd, 'vgg', a, b)
        v = ol.lpips(sd, 'vgg', a[None], b[None])
    assert u.shape == v.shape == (1, 1, 1, 1) and torch.equal(u, v)


@pytest.mark.parametrize('net,H,W', [('vgg', 37, 45), ('vgg', 16, 17), ('alex', 31, 33), ('alex', 257, 131)])
def test_odd_sizes_pool_with_floor(net, H, W):
    """Stage sizes follow floor((h - k) / s) + 1 at every pool; the restatement's stages have those shapes."""
    sd = ol.random_state_dict(net, seed=6)
    x = torch.rand(3, H, W, generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        st = ol.stages(sd, net, x)
    h, w = H, W
    for (kind, a, b), s in zip(ol.OPS[net], st[1:]):
        if kind == 'pool':
            h, w = (h - a) // b + 1, (w - a) // b + 1
        else:
            _, _, co, ks, stride, pad = ol.CONVS[net][a]
            h, w = (h + 2 * pad - ks) // stride + 1, (w + 2 * pad - ks) // stride + 1
        assert tuple(s.shape) == (1, s.shape[1], h, w)
    assert h >= 1 and w >= 1


def test_entry_points_validate_arguments_without_a_gpu():
    """A NULL output / parameter array / parameter, an unknown net and a wrong parameter count are
    K4_ERR_INVALID_ARG before any CUDA call; a NULL net has no workspace and no forward."""
    from k4nerf import _lib
    lib = _lib.lib
    buf = C.create_string_buffer(4096)
    p = C.addressof(buf)
    out = C.c_void_p()
    ptrs = (C.c_void_p * 31)(*([p] * 31))
    assert lib.k4_lpips_create(0, ptrs, 31, None, None) == K4_ERR_INVALID_ARG
    assert lib.k4_lpips_create(0, None, 31, None, C.byref(out)) == K4_ERR_INVALID_ARG
    for net, n in ((0, 30), (0, 15), (1, 31), (1, 14), (2, 31), (-1, 15)):
        assert lib.k4_lpips_create(net, ptrs, n, None, C.byref(out)) == K4_ERR_INVALID_ARG, (net, n)
    holes = (C.c_void_p * 31)(*([p] * 31))
    holes[17] = None
    assert lib.k4_lpips_create(0, holes, 31, None, C.byref(out)) == K4_ERR_INVALID_ARG
    assert out.value is None
    assert lib.k4_lpips_workspace_bytes(None, 64, 64) == 0
    st = (C.c_int64 * 3)(3 * 64, 3, 1)
    assert lib.k4_lpips_forward(None, p, p, st, st, 64, 64, p, p, 1 << 20, None) == K4_ERR_INVALID_ARG
    shape = (C.c_int64 * 3)()
    assert lib.k4_testing_lpips_stage(None, p, st, 64, 64, 0, None, shape, p, 1 << 20, None) == K4_ERR_INVALID_ARG
