"""LPIPS 0.1 restated in plain torch (test infrastructure only): what ``lpips.LPIPS(net='vgg' | 'alex',
version='0.1')(in0, in1, normalize=True)`` computes, as utils.rgb_lpips (lib/utils.py:137-149) calls it.  The ``lpips``
package is not needed; everything here follows its definition.

- Input: ``[3, H, W]`` (unbatched, as rgb_lpips passes it) or ``[N, 3, H, W]`` images in [0, 1];
  ``normalize=True`` maps them to ``2 x - 1``.
- ScalingLayer: ``(x - shift) / scale`` with the ``[1, 3, 1, 1]`` buffers ``scaling_layer.shift`` = (-.030, -.088,
  -.188) and ``scaling_layer.scale`` = (.458, .448, .450); they broadcast an unbatched input to ``[1, 3, H, W]``.
- Trunk: torchvision ``vgg16().features`` (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3; keys ``net.slice1.{0,2}``,
  ``net.slice2.{5,7}``, ``net.slice3.{10,12,14}``, ``net.slice4.{17,19,21}``, ``net.slice5.{24,26,28}``; 2x2 / 2 max-pools
  at 4, 9, 16, 23) or ``alexnet().features`` (ReLUs at 1, 4, 7, 9, 11; keys ``net.slice1.0``, ``net.slice2.3``,
  ``net.slice3.6``, ``net.slice4.8``, ``net.slice5.10``; conv0 11x11 / 4 / pad 2, conv3 5x5 / pad 2, others 3x3 / pad 1;
  3x3 / 2 max-pools at 2 and 5).  Pools use floor sizes.
- Head per tap k: ``f / (sqrt(sum_c f^2) + 1e-10)`` per pixel, ``(f0 - f1)^2``, the 1x1 ``lin{k}.model.1.weight``
  (``[1, C_k, 1, 1]``, no bias; the dropout before it is inactive in eval), the mean over the tap's pixels.
- Result: the sum of the five tap means, ``[N, 1, 1, 1]``.
"""
import torch
import torch.nn.functional as F

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
EPS = 1e-10

# (key, cin, cout, kernel, stride, pad) in trunk order
VGG_CONVS = [('net.slice1.0', 3, 64), ('net.slice1.2', 64, 64), ('net.slice2.5', 64, 128), ('net.slice2.7', 128, 128),
             ('net.slice3.10', 128, 256), ('net.slice3.12', 256, 256), ('net.slice3.14', 256, 256),
             ('net.slice4.17', 256, 512), ('net.slice4.19', 512, 512), ('net.slice4.21', 512, 512),
             ('net.slice5.24', 512, 512), ('net.slice5.26', 512, 512), ('net.slice5.28', 512, 512)]
VGG_CONVS = [(k, ci, co, 3, 1, 1) for k, ci, co in VGG_CONVS]
ALEX_CONVS = [('net.slice1.0', 3, 64, 11, 4, 2), ('net.slice2.3', 64, 192, 5, 1, 2), ('net.slice3.6', 192, 384, 3, 1, 1),
              ('net.slice4.8', 384, 256, 3, 1, 1), ('net.slice5.10', 256, 256, 3, 1, 1)]
CONVS = {'vgg': VGG_CONVS, 'alex': ALEX_CONVS}
TAP_CHANNELS = {'vgg': (64, 128, 256, 512, 512), 'alex': (64, 192, 384, 256, 256)}
# the trunk's operations in order: ('conv', index into CONVS[net], tap or None) or ('pool', kernel, stride)
OPS = {
    'vgg': [('conv', 0, None), ('conv', 1, 0), ('pool', 2, 2), ('conv', 2, None), ('conv', 3, 1), ('pool', 2, 2),
            ('conv', 4, None), ('conv', 5, None), ('conv', 6, 2), ('pool', 2, 2), ('conv', 7, None), ('conv', 8, None),
            ('conv', 9, 3), ('pool', 2, 2), ('conv', 10, None), ('conv', 11, None), ('conv', 12, 4)],
    'alex': [('conv', 0, 0), ('pool', 3, 2), ('conv', 1, 1), ('pool', 3, 2), ('conv', 2, 2), ('conv', 3, 3), ('conv', 4, 4)],
}


def param_keys(net):
    """The parameters in the C ABI's order (k4_lpips_create): every convolution's weight and bias in trunk order,
    then lin0 .. lin4."""
    keys = []
    for k, *_ in CONVS[net]:
        keys += [k + '.weight', k + '.bias']
    return keys + [f'lin{i}.model.1.weight' for i in range(5)]


def param_shapes(net):
    shapes = {}
    for k, ci, co, ks, _, _ in CONVS[net]:
        shapes[k + '.weight'] = (co, ci, ks, ks)
        shapes[k + '.bias'] = (co,)
    for i, c in enumerate(TAP_CHANNELS[net]):
        shapes[f'lin{i}.model.1.weight'] = (1, c, 1, 1)
    return shapes


def random_state_dict(net, seed=0):
    """Seeded fp32 parameters of the real shapes: He-scaled convolutions (so that activations neither vanish nor blow
    up through the trunk), small biases, non-negative lin weights (as trained LPIPS heads are), and the scaling layer."""
    g = torch.Generator().manual_seed(seed)
    sd = {'scaling_layer.shift': torch.tensor(SHIFT).view(1, 3, 1, 1), 'scaling_layer.scale': torch.tensor(SCALE).view(1, 3, 1, 1)}
    for k, shape in param_shapes(net).items():
        if k.endswith('.bias'):
            sd[k] = 0.05 * torch.randn(shape, generator=g)
        elif k.startswith('lin'):
            sd[k] = torch.rand(shape, generator=g) * (2.0 / shape[1])
        else:
            fan_in = shape[1] * shape[2] * shape[3]
            sd[k] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
    return sd


def scale_input(x, dtype=torch.float64):
    """normalize=True and the ScalingLayer: ``[3, H, W]`` -> ``[1, 3, H, W]`` (the buffers' broadcast)."""
    x = x.to(dtype)
    shift = torch.tensor(SHIFT, dtype=torch.float32).to(dtype).view(1, 3, 1, 1).to(x.device)
    scale = torch.tensor(SCALE, dtype=torch.float32).to(dtype).view(1, 3, 1, 1).to(x.device)
    return (2 * x - 1 - shift) / scale


def op(sd, net, i, x):
    """Operation i of the trunk on x ([N, C, h, w])."""
    kind, a, b = OPS[net][i]
    if kind == 'pool':
        return F.max_pool2d(x, a, b)
    k, _, _, _, stride, pad = CONVS[net][a]
    w, bias = sd[k + '.weight'].to(x), sd[k + '.bias'].to(x)
    return F.relu(F.conv2d(x, w, bias, stride=stride, padding=pad))


def stages(sd, net, x, dtype=torch.float64):
    """[scaled input, output of op 1, ..., output of the last op] for one image."""
    out = [scale_input(x, dtype)]
    for i in range(len(OPS[net])):
        out.append(op(sd, net, i, out[-1]))
    return out


def taps(sd, net, x, dtype=torch.float64):
    st = stages(sd, net, x, dtype)
    return [st[i + 1] for i, (kind, _, t) in enumerate(OPS[net]) if kind == 'conv' and t is not None]


def head(sd, k, f0, f1):
    """Tap k's term: the spatial mean of lin_k((f0 / (|f0| + eps) - f1 / (|f1| + eps))^2), [N, 1, 1, 1]."""
    n0 = f0 / (torch.sqrt(torch.sum(f0 ** 2, dim=1, keepdim=True)) + EPS)
    n1 = f1 / (torch.sqrt(torch.sum(f1 ** 2, dim=1, keepdim=True)) + EPS)
    d = F.conv2d((n0 - n1) ** 2, sd[f'lin{k}.model.1.weight'].to(f0))
    return d.mean([2, 3], keepdim=True)


def lpips(sd, net, in0, in1, dtype=torch.float64):
    """The LPIPS score of in0, in1 ([3, H, W] or [N, 3, H, W] in [0, 1]) in ``dtype``: ``[N, 1, 1, 1]``.  Both images
    go through the trunk in lockstep and each tap's term is formed as soon as it exists, so that only the current
    activations are held (a 4032 x 3024 pair in fp64 fits on one GPU)."""
    x0, x1 = scale_input(in0, dtype), scale_input(in1, dtype)
    val = None
    for i, (kind, _, t) in enumerate(OPS[net]):
        x0, x1 = op(sd, net, i, x0), op(sd, net, i, x1)
        if kind == 'conv' and t is not None:
            h = head(sd, t, x0, x1)
            val = h if val is None else val + h
    return val


def macs(net, H, W):
    """Multiply-accumulates of one image's trunk at H x W (from the layer shapes)."""
    total, h, w = 0, H, W
    for kind, a, b in OPS[net]:
        if kind == 'pool':
            h, w = (h - a) // b + 1, (w - a) // b + 1
            continue
        _, ci, co, ks, s, p = CONVS[net][a]
        h, w = (h + 2 * p - ks) // s + 1, (w + 2 * p - ks) // s + 1
        total += h * w * co * ci * ks * ks
    return total
