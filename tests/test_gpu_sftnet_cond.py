"""GPU: the view-conditioned VC-Decoder, SFTNet(3, 4, 64, n, 32, num_cond) with a condition of up to 64 channels.  CondNet
element by element through k4_testing_condnet with the tensor-core kernel (condnet_wide_mma_kernel) and the fp32 kernel
forced; the whole net against golden vectors of the REFERENCE's own module (tests/golden/make_golden_cond.py) and against
cuDNN in true fp32; row windows and peer destinations; render_frame_4k; and a depth decoder in the same process."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import k4nerf
from k4nerf import _lib, render
from k4nerf.sr_esrnet import sft_condition
from oracle import pipeline, scenes, sftnet
from helpers import make_state, model_from_state
from test_gpu_sr_layers import (FP16_MAX, GAMMA_TC, U, check_condnet_outputs, depth_map, hwc, lrelu, sm_count,
                                _sft_ptrs, _stream)
from test_sftnet_cond import frame_condition, golden_inputs, pretrained_cond64_state_dict, pretrained_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MMA, FP32 = _lib.K4_SR_KERNEL_MMA, _lib.K4_SR_KERNEL_FP32
PKNAME = {_lib.K4_SR_KERNEL_AUTO: 'auto', MMA: 'mma', FP32: 'fp32'}
SENT16, SENT32 = -7.0, -7.25


# ------------------------------------------------------------------------------------------------
# CondNet with a wide condition, element by element
# ------------------------------------------------------------------------------------------------
def condnet_params(nc, seed, dev, scale=1.0):
    """CondNet.0 (64 x nc x 3x3), .2, .4 (64x64), .6 (32x64), weight and bias each, nn.Conv2d's uniform initialisation
    (+-1 / sqrt(fan_in)) times `scale`."""
    g = torch.Generator().manual_seed(seed)
    ts = []
    for shape, fan in (((64, nc, 3, 3), 9 * nc), ((64, 64, 1, 1), 64), ((64, 64, 1, 1), 64), ((32, 64, 1, 1), 64)):
        bound = scale / math.sqrt(fan)
        ts += [(torch.rand(shape, generator=g) * 2 - 1) * bound, (torch.rand(shape[0], generator=g) * 2 - 1) * bound]
    return [t.contiguous().to(dev) for t in ts]


def cond_map(nc, H, W, seed, dev):
    """[nc, H, W]: run_sr.py's conditions for 63 / 64 (the view embedding, whose high frequencies change sign from pixel
    to pixel, behind a depth map for 64); for other widths a depth-like channel and uniform noise in [-1, 1]."""
    if nc in (63, 64):
        return frame_condition(nc, H, W, seed).to(dev)
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(nc, H, W, generator=g) * 2 - 1
    c[0] = depth_map(H, W, seed + 1, 'cpu')
    return c.contiguous().to(dev)


def run_condnet(params, cond_in, kernel, rows=None):
    nc, H, W = cond_in.shape
    out = torch.full((H * W, 32), SENT32, device=cond_in.device)
    c16 = torch.full((H * W, 32), SENT16, dtype=torch.float16, device=cond_in.device)
    a = _lib.CondnetTestArgs()
    a.h_condnet = _sft_ptrs(params)
    a.d_cond_in, a.H, a.W, a.num_cond = cond_in.data_ptr(), H, W, nc
    a.y_lo, a.y_hi = rows if rows is not None else (0, H)
    a.d_cond_out, a.d_cond16, a.kernel = out.data_ptr(), c16.data_ptr(), kernel
    used = C.c_int32(-9)
    st = _lib.lib.k4_testing_condnet(C.byref(a), C.byref(used), _stream())
    assert st == 0, f'k4_testing_condnet -> {st} ({_lib.lib.k4_status_string(st).decode()}) for {PKNAME[kernel]}'
    if kernel != _lib.K4_SR_KERNEL_AUTO:
        assert used.value == kernel, (PKNAME[kernel], used.value)
    return out, c16, used.value


def condnet_ref(p, cond_in, kernel):
    """fp64 CondNet of a [nc, H, W] condition with the per-element bound E of `kernel` carried layer to layer, as
    test_gpu_sr_layers.condnet_ref does for the depth condition; only layer 0 differs.  Its 9 nc products are summed in
    chunks, in the kernel's order, from the bias; every rounding of chunk k is bounded through |P_{k-1}| + S_k, the
    partial sum before the chunk (fp64) plus the chunk's sum of |products| -- 576 products of sign-changing operands
    cancel, so |P| stays far below the whole reduction's S:
      * fp32 kernel: one chunk per channel, 9 FFMAs each within u (|P_{k-1}| + S_k).
      * mma kernel: one chunk per tap and k16 step (taps row-major, channels 16 ks .. 16 ks + 15), 3 MMA instructions of
        17 * 2^-23 (|P_{k-1}| + S_k) each, on split operands -- the condition a = ah + al and the weights w = wh + wl,
        |x - hi - lo| <= 2^-22 |x| + 2^-25 and |lo| <= 2^-11 |x| + 2^-24 -- whose dropped al wl term and representation
        errors are added as for the 1x1 layers (taps outside the map are exact zeros).
    Returns the output [P, 32], the bound [P, 32] and the largest |hidden activation|."""
    nc = cond_in.shape[0]
    W0, b0 = p[0].double(), p[1].double()
    c = cond_in.double()[None]
    conv = lambda a, w: hwc(F.conv2d(a, w, padding=1)[0])
    z = hwc(F.conv2d(c, W0, b0, padding=1)[0])
    av, aw = c.abs(), W0.abs()
    if kernel == FP32:
        chunks = [(ci, slice(None), slice(None)) for ci in range(nc)]
        S_of, n_round, gamma = (lambda m: conv(av, aw * m)), 9, U
    else:
        ev, lv = 2.0 ** -22 * av + 2.0 ** -25, 2.0 ** -11 * av + 2.0 ** -24
        ew, lw = 2.0 ** -22 * aw + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -24
        chunks = [(slice(16 * ks, 16 * ks + 16), t // 3, t % 3) for t in range(9) for ks in range((nc + 15) // 16)]
        S_of, n_round, gamma = (lambda m: conv(av, aw * m) + conv(av, lw * m) + conv(lv, aw * m)), 3, GAMMA_TC
    P = b0.expand_as(z).clone()
    acc = torch.zeros_like(z)
    for ch in chunks:
        m = torch.zeros_like(W0)
        m[(slice(None),) + ch] = 1.0
        acc += n_round * (P.abs() + S_of(m))
        P += conv(c, W0 * m)
    E = 1.01 * gamma * acc
    if kernel != FP32:
        E = E + conv(lv, lw) + conv(av, ew) + conv(ev, aw) + conv(ev, ew)
    hmax = 0.0
    for i in (2, 4, 6):
        a = lrelu(z)
        D = E + 2 * U * (z.abs() + E)
        hmax = max(hmax, a.abs().max().item())
        Wl, bl = p[i].double().view(p[i].shape[0], 64), p[i + 1].double()
        av, aw = a.abs() + D, Wl.abs()
        z = a @ Wl.T + bl
        if kernel == FP32:
            E = D @ aw.T + 65 * U * (av @ aw.T + bl.abs())
        else:
            ev, lv = 2.0 ** -22 * av + 2.0 ** -25, 2.0 ** -11 * av + 2.0 ** -24
            ew, lw = 2.0 ** -22 * aw + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -24
            split = lv @ lw.T + av @ ew.T + ev @ aw.T + ev @ ew.T
            S = av @ aw.T + av @ lw.T + lv @ aw.T + bl.abs()
            E = D @ aw.T + split + 12 * GAMMA_TC * S
    return z, E, hmax


WIDE_CASES = [  # (name, H, W, rows, weight scale)
    ('1x1', 1, 1, None, 1.0), ('1x7', 1, 7, None, 1.0), ('7x1', 7, 1, None, 4.0), ('19x13', 19, 13, None, 1.0),
    ('19x13_w4', 19, 13, None, 4.0), ('rows5-6', 40, 29, (5, 6), 1.0), ('rows3-37', 40, 29, (3, 37), 4.0),
    ('rows16-33', 40, 29, (16, 33), 1.0),
]


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
@pytest.mark.parametrize('nc', (5, 63, 64))
@pytest.mark.parametrize('case', WIDE_CASES, ids=lambda c: c[0])
def test_wide_condnet_meets_its_element_bound(case, nc, kernel, cuda_device):
    """Shapes down to 1x1, P = 247 (not a multiple of 16) and row windows strictly inside the map, whose edge rows must see
    the real neighbour rows: every output within the bound of condnet_ref, cond16 the saturated fp16 rounding of
    cond_out, rows outside the window untouched."""
    name, H, W, rows, scale = case
    p = condnet_params(nc, 200 + H + W + nc, 'cuda', scale)
    cond_in = cond_map(nc, H, W, 300 + H + nc, 'cuda')
    ref, E, _ = condnet_ref(p, cond_in, kernel)
    out, c16, _ = run_condnet(p, cond_in, kernel, rows)
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, E, rows, H, W, f'wide condnet nc={nc} {name} ({PKNAME[kernel]})')


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
def test_wide_condnet_grid_stride_wraps(kernel, cuda_device):
    """More than 3 x (SM-count CTAs x 8 warps x 16 pixels): the wide mma kernel's grid of one CTA per SM strides over
    the map more than three times."""
    W = 331
    H = 3 * sm_count() * 8 * 16 // W + 3
    assert H * W > 3 * sm_count() * 8 * 16
    p = condnet_params(64, 400, 'cuda')
    cond_in = cond_map(64, H, W, 401, 'cuda')
    ref, E, _ = condnet_ref(p, cond_in, kernel)
    out, c16, _ = run_condnet(p, cond_in, kernel, (1, H))
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, E, (1, H), H, W, f'wide condnet {H}x{W} ({PKNAME[kernel]})')


def exact_wide_operands(nc, H, W, seed, dev):
    """Non-negative operands whose every product and sum is exact in fp32 and whose every split operand fits hi + lo
    exactly, with no lo x lo product: channels below nc / 2 carry 12-bit condition values ((2^11 + odd) 2^-15, an fp16
    lo part each) and meet CondNet.0 weights j/8; channels from nc / 2 on carry values on the 1/2 grid and meet 12-bit
    weights ((2^11 + odd) 2^-16).  Each output of layer 0 has 9 non-zero weights; CondNet.2, .4, .6 rows have two
    weights of 1/2; biases m/64."""
    g = torch.Generator().manual_seed(seed)
    h = nc // 2
    cond = torch.empty(nc, H, W)
    cond[:h] = (2 ** 11 + 2 * torch.randint(0, 2 ** 10, (h, H, W), generator=g) + 1) * 2.0 ** -15
    cond[h:] = torch.randint(0, 3, (nc - h, H, W), generator=g) / 2.0
    w0 = torch.zeros(64, nc * 9)
    for o in range(64):
        for k in torch.randperm(nc * 9, generator=g)[:9].tolist():
            w0[o, k] = (torch.randint(0, 3, (1,), generator=g).item() / 8.0 if k // 9 < h else
                        (2 ** 11 + 2 * torch.randint(0, 2 ** 10, (1,), generator=g).item() + 1) * 2.0 ** -16)

    def sparse(n_out):
        w = torch.zeros(n_out, 64)
        for o in range(n_out):
            w[o, torch.randperm(64, generator=g)[:2]] = 0.5
        return w.view(n_out, 64, 1, 1)

    bias = lambda n: torch.randint(0, 17, (n,), generator=g) / 64.0
    ts = [w0.view(64, nc, 3, 3), bias(64), sparse(64), bias(64), sparse(64), bias(64), sparse(32), bias(32)]
    return [t.contiguous().to(dev) for t in ts], cond.contiguous().to(dev)


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
@pytest.mark.parametrize('nc', (5, 63, 64))
def test_wide_condnet_exact_operands(nc, kernel, cuda_device):
    """Both kernels EQUAL the fp64 reference on exact operands: a lost condition lo term (al * Wh) or weight lo term
    (ah * Wl) of layer 0, a moved tap or channel, or a wrong padding row is a non-zero difference."""
    H, W = 23, 37
    p, cond_in = exact_wide_operands(nc, H, W, 500 + nc, 'cuda')
    ref, _, _ = condnet_ref(p, cond_in, kernel)
    c = cond_in.double()
    assert bool(((c - c.half().double()) != 0).any()), 'no condition lo part: the case lost its point'
    w0 = p[0].double()
    assert bool(((w0 - w0.half().double()) != 0).any()), 'no weight lo part: the case lost its point'
    z = hwc(F.conv2d(c[None], w0, p[1].double(), padding=1)[0])
    for i in (2, 4, 6):
        assert torch.equal(z.float().double(), z), 'a sum is not exact in fp32'
        hi = z.half().double()
        assert torch.equal((z - hi).half().double(), z - hi), 'an activation does not fit the hi + lo split'
        z = z @ p[i].double().view(-1, 64).T + p[i + 1].double()
    assert torch.equal(z.float().double(), z)
    rows = (3, 20)
    out, c16, _ = run_condnet(p, cond_in, kernel, rows)
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, None, rows, H, W, f'wide condnet exact nc={nc} ({PKNAME[kernel]})')


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
def test_wide_condnet_huge_inputs_stay_finite(kernel, cuda_device):
    """Condition values of 1e6 (beyond fp16: the mma kernel's hi and lo parts both saturate) and CondNet.0 scaled by 2^10:
    every output finite, cond16 the saturated rounding of cond_out."""
    H, W = 19, 13
    p = condnet_params(64, 600, 'cuda')
    p[0] = p[0] * 2.0 ** 10
    cond_in = cond_map(64, H, W, 601, 'cuda')
    cond_in[0, ::3] = 1e6
    cond_in[7, :, ::2] = -1e6
    _, _, hmax = condnet_ref(p, cond_in, kernel)
    assert hmax > 2 * FP16_MAX, 'the case lost its point'
    out, c16, _ = run_condnet(p, cond_in, kernel)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(c16).all()
    assert torch.equal(c16.view(torch.int16), out.clamp(-FP16_MAX, FP16_MAX).half().view(torch.int16))


def test_condnet_auto_follows_the_env_switch_for_a_wide_condition(monkeypatch, cuda_device):
    p = condnet_params(63, 610, 'cuda')
    cond_in = cond_map(63, 5, 9, 611, 'cuda')
    monkeypatch.delenv('K4_CONDNET_FP32', raising=False)
    assert run_condnet(p, cond_in, _lib.K4_SR_KERNEL_AUTO)[2] == MMA
    monkeypatch.setenv('K4_CONDNET_FP32', '1')
    assert run_condnet(p, cond_in, _lib.K4_SR_KERNEL_AUTO)[2] == FP32


# ------------------------------------------------------------------------------------------------
# the whole net
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', params=(63, 64))
def net(request, cuda_device):
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, request.param)
    n.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=request.param))
    return n.to(cuda_device)


def test_cond_forward_and_tile_process_match_reference_golden(net, cuda_device):
    nc = net.num_cond
    gold = torch.load(os.path.join(GOLD, f'sftnet_cond{nc}_ref.pt'), map_location='cpu', weights_only=False)
    x, c, xt, ct = golden_inputs(nc)
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    assert y.shape == gold['forward'].shape == (1, 3, 80, 112)
    p = pipeline.psnr(y, gold['forward'])
    yt = net.tile_process(xt.to(cuda_device), ct.to(cuda_device), tile_size=16, tile_pad=10)
    assert yt.device.type == 'cpu' and yt.shape == gold['tile_process'].shape == (1, 3, 96, 160)
    pt = pipeline.psnr(yt, gold['tile_process'])
    print(f'num_cond {nc}: forward {p:.2f} dB, tile_process {pt:.2f} dB vs the reference module')
    assert p >= 65.0 and pt >= 65.0, (p, pt)


@pytest.fixture(scope='module')
def net_pretrained(cuda_device):
    sd = pretrained_cond64_state_dict()
    if sd is None:
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing (python oracle/build_ref.py where /root/reference exists)')
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, 64)
    n.load_state_dict(sd)
    return n.to(cuda_device), {k: v.to(cuda_device) for k, v in sd.items()}


def _fp32_and_tf32(fn):
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
        a = fn()
        torch.backends.cudnn.allow_tf32 = True; torch.backends.cuda.matmul.allow_tf32 = True
        b = fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return a, b


def test_cond64_pretrained_forward_matches_reference_module_golden(net_pretrained, cuda_device):
    net, _ = net_pretrained
    gold = torch.load(os.path.join(GOLD, 'sftnet_cond64_pretrained_ref.pt'), map_location='cpu', weights_only=False)
    x, c = pretrained_inputs()
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    p = pipeline.psnr(y, gold['forward'])
    print('pretrained num_cond 64 vs reference-module golden: PSNR', p, 'maxabs', (y - gold['forward']).abs().max().item())
    assert p >= 65.0, p


def test_cond64_pretrained_520_tile_vs_cudnn_fp32(net_pretrained, cuda_device):
    net, sd = net_pretrained
    g = torch.Generator().manual_seed(36)
    x = (torch.rand(1, 3, 520, 520, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = frame_condition(64, 520, 520, 37)[None].to(cuda_device)
    ref32, ref_tf32 = _fp32_and_tf32(lambda: sftnet.sftnet_forward(sd, x, c))
    y = net(x, c)
    p, p_tf32 = pipeline.psnr(y.cpu(), ref32.cpu()), pipeline.psnr(ref_tf32.cpu(), ref32.cpu())
    print(f'num_cond 64, 520x520 tile, pretrained weights: k4nerf vs cuDNN fp32 {p:.2f} dB; cuDNN TF32 vs fp32 {p_tf32:.2f} dB')
    assert y.shape == (1, 3, 2080, 2080)
    assert p >= 65.0, (p, p_tf32)


def test_cond64_pretrained_full_frame_tile_process_vs_cudnn_fp32(net_pretrained, cuda_device):
    """1008x756 -> 4032x3024, tile 510 / pad 10, with the 3-D [64, H, W] condition of the reference's contract."""
    net, sd = net_pretrained
    g = torch.Generator().manual_seed(38)
    x = (torch.rand(1, 3, 756, 1008, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = frame_condition(64, 756, 1008, 39).to(cuda_device)
    ref32, ref_tf32 = _fp32_and_tf32(lambda: sftnet.tile_process(sd, x, c, 510, 10))
    y = net.tile_process(x, c, 510, 10)
    assert y.shape == (1, 3, 3024, 4032) and y.device.type == 'cpu'
    p, p_tf32 = pipeline.psnr(y, ref32), pipeline.psnr(ref_tf32, ref32)
    print(f'num_cond 64, 1008x756 tile_process(510), pretrained: k4nerf vs cuDNN fp32 {p:.2f} dB; TF32 vs fp32 {p_tf32:.2f} dB')
    assert p >= 65.0, (p, p_tf32)


def test_cond_forward_roi_block_is_bit_identical_to_the_full_forward(net, cuda_device):
    h, w = 210, 44
    g = torch.Generator().manual_seed(41)
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = frame_condition(net.num_cond, h, w, 42)[None].to(cuda_device)
    full = net(x, c)
    frame = torch.full((3, 4 * h + 8, 4 * w + 12), -7.0, device=cuda_device)
    for keep in ((0, h, 0, w), (0, 100, 0, w), (101, 131, 3, 40), (180, h, 10, w), (95, 96, 0, 1)):
        y0, y1, x0, x1 = keep
        frame.fill_(-7.0)
        dst = frame[:, 4:4 + 4 * (y1 - y0), 8:8 + 4 * (x1 - x0)]
        net.forward_roi(x, c, keep, dst)
        assert torch.equal(dst, full[0, :, 4 * y0:4 * y1, 4 * x0:4 * x1]), keep
        dst.fill_(-7.0)
        assert bool((frame == -7.0).all()), ('wrote outside the destination window', keep)


@pytest.mark.parametrize('world', [2, 3, 5, 8])
def test_cond_row_parts_with_halo_reproduce_the_unsplit_tile(net, cuda_device, world):
    from k4nerf import dist as kdist
    assert net.receptive_halo() == 80
    H, W = 300, 40
    g = torch.Generator().manual_seed(21)
    x = (torch.rand(1, 3, H, W, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = frame_condition(net.num_cond, H, W, 22).to(cuda_device)
    ref = net.tile_process(x, c, tile_size=510, tile_pad=10, to_cpu=False)
    units = kdist.sr_units(H, W, 510, 10, world, net.receptive_halo())
    assert len(units) == world
    out = torch.zeros_like(ref)
    for u in units:
        sa, sb, xa, xb = u['src']
        assert sb - sa < H
        o = net(x[:, :, sa:sb, xa:xb], c.unsqueeze(0)[:, :, sa:sb, xa:xb])
        ky, kx = u['keep']
        y0, y1, x0, x1 = u['dst']
        out[:, :, 4 * y0:4 * y1, 4 * x0:4 * x1] = o[:, :, 4 * ky:4 * (ky + y1 - y0), 4 * kx:4 * (kx + x1 - x0)]
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    assert torch.equal(net.tile_process_sharded(x, c, tile_size=510, tile_pad=10), ref)


def test_cond_forward_roi_extra_destinations_receive_the_same_block(net, cuda_device):
    h, w = 96, 52
    g = torch.Generator().manual_seed(43)
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = frame_condition(net.num_cond, h, w, 44)[None].to(cuda_device)
    full = net(x, c)
    frames = [torch.full((3, 4 * h, 4 * w), -7.0, device=cuda_device) for _ in range(3)]
    for keep in ((0, h, 0, w), (10, 61, 3, 40)):
        y0, y1, x0, x1 = keep
        for f in frames:
            f.fill_(-7.0)
        win = lambda f: f[:, 4 * y0:4 * y1, 4 * x0:4 * x1]
        dst = win(frames[0])
        net.forward_roi(x, c, keep, dst, extra=[f.data_ptr() + 4 * dst.storage_offset() for f in frames[1:]])
        for f in frames:
            assert torch.equal(win(f), full[0, :, 4 * y0:4 * y1, 4 * x0:4 * x1]), keep
            chk = f.clone()
            win(chk).fill_(-7.0)
            assert bool((chk == -7.0).all()), ('wrote outside the destination window', keep)


_CHILD = r'''
import sys
import torch
sys.path[:0] = [sys.argv[1], sys.argv[1] + '/4k-nerf_b200', sys.argv[1] + '/tests']
import k4nerf
from oracle import sftnet
from test_sftnet_cond import frame_condition
nc = int(sys.argv[3])
n = k4nerf.SFTNet(3, 4, 64, 5, 32, nc)
n.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=nc))
n = n.cuda()
g = torch.Generator().manual_seed(5)
x = torch.rand(1, 3, 19, 13, generator=g)
c = frame_condition(nc, 19, 13, 6)[None]
torch.save(n(x.cuda(), c.cuda()).cpu(), sys.argv[2])
'''


@pytest.mark.parametrize('nc', (63, 64))
def test_cond_condnet_fp32_switch_in_child_processes(nc, tmp_path, cuda_device):
    """K4_CONDNET_FP32=1 runs the fp32 CondNet of a wide condition in the decoder: both runs reach 60 dB against
    oracle.sftnet and agree with each other within the bar of the existing switches (66 dB)."""
    base = {k: v for k, v in os.environ.items() if not k.startswith('K4_')}
    flags = ['-s'] if sys.flags.no_user_site else []
    outs = {}
    for name, env in (('default', {}), ('condnet_fp32', {'K4_CONDNET_FP32': '1'})):
        path = tmp_path / f'{name}.pt'
        r = subprocess.run([sys.executable, *flags, '-c', _CHILD, ROOT, str(path), str(nc)], env=dict(base, **env),
                           cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (name, r.stderr[-3000:])
        outs[name] = torch.load(path)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1, 3, 19, 13, generator=g)
    ref = sftnet.sftnet_forward(sftnet.random_state_dict(seed=3, num_cond=nc), x, frame_condition(nc, 19, 13, 6)[None])
    for name, y in outs.items():
        p, pd = pipeline.psnr(y, ref), pipeline.psnr(y, outs['default'])
        print(f'num_cond {nc} {name}: {p:.2f} dB vs oracle, {pd:.2f} dB vs default')
        assert p >= 60.0, (name, p)
        assert name == 'default' or pd >= 66.0, (name, pd)


def test_render_frame_4k_with_a_view_conditioned_decoder(net, cuda_device):
    """render_frame_4k builds the condition from the LR frame's depth and viewdirs: equal to the marcher, then
    sft_condition, then tile_process."""
    dev = cuda_device
    nc = net.num_cond
    st = make_state('cfgA', res=32, regime='fog')
    m = model_from_state(st, dev)
    H, W = 20, 28
    K, c2w = scenes.blender_camera(H, W)
    kw = dict(scenes.RENDER_KW_DVGO)
    sr, lr = render.render_frame_4k(m, net, H, W, K, c2w, False, kw, test_tile=16)
    assert sr.shape == (3, 4 * H, 4 * W) and sr.is_cuda
    _, depths, _, _, viewdirs, feats = render.render_viewpoints_sr(m, np.array([c2w.numpy()]), np.array([[H, W]]),
                                                                    np.array([K]), False, kw)
    x = torch.from_numpy(feats[0]).movedim(-1, 0).unsqueeze(0).to(dev)
    depth = torch.from_numpy(depths[0]).to(dev)
    cond = sft_condition(nc, depth, viewdirs[0], H, W)
    assert cond.shape == (nc, H, W)
    ref = net.tile_process(x, cond, tile_size=16).squeeze(0).clamp(0, 1)
    assert (sr.cpu() - ref).abs().max().item() < 2e-3
    # the sharded form in a single process: its one rank generates the frame's viewdirs itself
    srs, _ = render.render_frame_4k_sharded(m, net, H, W, K, c2w, False, kw, test_tile=16)
    assert torch.equal(srs, sr)


_DEPTH_SCRIPT = r'''
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import torch
import k4nerf
from oracle import sftnet
dev = torch.device('cuda', 0)
n = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
n.load_state_dict(sftnet.random_state_dict(seed=3))
n = n.to(dev)
g = torch.Generator().manual_seed(61)
x = (torch.rand(1, 3, 45, 70, generator=g) * 1.2 - 0.1).to(dev)
c = torch.rand(1, 45, 70, generator=g).to(dev)
torch.save(n.tile_process(x, c, 32, 10).cpu(), {out!r})
'''


def test_depth_decoder_after_a_64_channel_decoder_matches_a_fresh_process(cuda_device, tmp_path):
    """No launcher state of the wide CondNet leaks into the depth decoder: a num_cond = 1 net built and run after a 64
    one in this process decodes bit for bit what it decodes in a fresh interpreter."""
    n64 = k4nerf.SFTNet(3, 4, 64, 5, 32, 64)
    n64.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=64))
    n64 = n64.to(cuda_device)
    g = torch.Generator().manual_seed(61)
    x = (torch.rand(1, 3, 45, 70, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 45, 70, generator=g).to(cuda_device)
    y64 = n64.tile_process(x, frame_condition(64, 45, 70, 62).to(cuda_device), 32, 10)
    assert y64.shape == (1, 3, 180, 280) and torch.isfinite(y64).all()
    n1 = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    n1.load_state_dict(sftnet.random_state_dict(seed=3))
    here = n1.to(cuda_device).tile_process(x, c, 32, 10)
    out = str(tmp_path / 'depth.pt')
    code = _DEPTH_SCRIPT.format(root=ROOT, pkg=os.path.join(ROOT, '4k-nerf_b200'), out=out)
    subprocess.run([sys.executable, '-c', code], check=True, timeout=600)
    fresh = torch.load(out, map_location='cpu', weights_only=False)
    assert here.shape == fresh.shape == (1, 3, 180, 280)
    assert torch.equal(here, fresh)
