"""GPU: the x1 VC-Decoder, SFTNet(3, 1, 64, 5, 32, 1) of the reference's 1x configurations, through the C ABI.
The body is the x4 decoder's; the tail is conv_hr + LeakyReLU and conv_last at the input resolution, and the output
has the input's size.  Against golden vectors of the REFERENCE's own module at scale 1 (tests/golden/make_golden_x1.py)
and the functional oracle, plus the row windows, the C-ABI contract of the scale and the independence of x1 and x4
nets in one process."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import k4nerf
from k4nerf import _lib, render
from oracle import pipeline, scenes, sftnet
from helpers import make_state, model_from_state
from test_sftnet_x1 import pretrained_x1_state_dict, x1_state_dict

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K4_ERR_INVALID_ARG, K4_ERR_UNSUPPORTED, K4_ERR_WORKSPACE = -1, -2, -4


def _inputs():
    g = torch.Generator().manual_seed(11)
    x = torch.rand(1, 3, 20, 28, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, 20, 28, generator=g)
    xt = torch.rand(1, 3, 24, 40, generator=g) * 1.2 - 0.1
    ct = torch.rand(1, 24, 40, generator=g)
    return x, c, xt, ct


@pytest.fixture(scope='module')
def net(cuda_device):
    n = k4nerf.SFTNet(3, 1, 64, 5, 32, 1)
    n.load_state_dict(x1_state_dict(seed=3))
    return n.to(cuda_device)


def test_x1_forward_matches_reference_golden(net, cuda_device):
    gold = torch.load(os.path.join(GOLD, 'sftnet_x1_ref.pt'), map_location='cpu', weights_only=False)
    x, c, _, _ = _inputs()
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    assert y.shape == gold['forward'].shape == (1, 3, 20, 28)
    p = pipeline.psnr(y, gold['forward'])
    print('x1 SFTNet forward PSNR vs reference', p, 'maxabs', (y - gold['forward']).abs().max().item())
    assert p >= 65.0, p


def test_x1_tile_process_matches_reference_golden(net, cuda_device):
    gold = torch.load(os.path.join(GOLD, 'sftnet_x1_ref.pt'), map_location='cpu', weights_only=False)
    _, _, xt, ct = _inputs()
    y = net.tile_process(xt.to(cuda_device), ct.to(cuda_device), tile_size=16, tile_pad=10)
    assert y.device.type == 'cpu' and y.shape == gold['tile_process'].shape == (1, 3, 24, 40)
    p = pipeline.psnr(y, gold['tile_process'])
    print('x1 SFTNet tile_process PSNR vs reference', p)
    assert p >= 65.0, p


@pytest.mark.parametrize('hw', [(19, 13), (1, 7), (33, 50), (8, 8)])
def test_x1_ragged_sizes_match_oracle(net, cuda_device, hw):
    """Sizes that are not multiples of the 16x8 pixel tile, down to a single row; at x1 conv_last runs on that grid."""
    h, w = hw
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1, 3, h, w, generator=g)
    c = torch.rand(1, 1, h, w, generator=g)
    ref = sftnet.sftnet_forward(x1_state_dict(seed=3), x, c, scale=1)
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    assert y.shape == (1, 3, h, w)
    p = pipeline.psnr(y, ref)
    print('x1 ragged', hw, p)
    assert p >= 60.0, (hw, p)


# ------------------------------------------------------------------------------------------------
# real weights, real sizes: RealESRNet_x4plus.pth loaded strict=False into the x1 net as run_sr.py:663 does (conv_up1 /
# conv_up2 dropped), against the reference module's golden and against oracle.sftnet on cuDNN in true fp32 (TF32 off).
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def net_pretrained(cuda_device):
    sd = pretrained_x1_state_dict()
    if sd is None:
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing (python oracle/build_ref.py where /root/reference exists)')
    n = k4nerf.SFTNet(3, 1, 64, 5, 32, 1)
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


def test_x1_pretrained_forward_matches_reference_module_golden(net_pretrained, cuda_device):
    net, _ = net_pretrained
    gold = torch.load(os.path.join(GOLD, 'sftnet_x1_pretrained_ref.pt'), map_location='cpu', weights_only=False)
    g = torch.Generator().manual_seed(gold['input_seed'])
    x = torch.rand(1, 3, 40, 48, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, 40, 48, generator=g)
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    p = pipeline.psnr(y, gold['forward'])
    print('pretrained x1 SFTNet vs reference-module golden: PSNR', p, 'maxabs', (y - gold['forward']).abs().max().item())
    assert p >= 65.0, p


def test_x1_pretrained_520_tile_vs_cudnn_fp32(net_pretrained, cuda_device):
    net, sd = net_pretrained
    g = torch.Generator().manual_seed(31)
    x = (torch.rand(1, 3, 520, 520, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, 520, 520, generator=g).to(cuda_device)
    ref32, ref_tf32 = _fp32_and_tf32(lambda: sftnet.sftnet_forward(sd, x, c, scale=1))
    y = net(x, c)
    p, p_tf32 = pipeline.psnr(y.cpu(), ref32.cpu()), pipeline.psnr(ref_tf32.cpu(), ref32.cpu())
    print(f'x1 520x520 tile, pretrained weights: k4nerf vs cuDNN fp32 {p:.2f} dB (maxabs {(y - ref32).abs().max().item():.3e}); '
          f'cuDNN TF32 (the reference default) vs cuDNN fp32 {p_tf32:.2f} dB')
    assert y.shape == (1, 3, 520, 520)
    assert p >= 65.0, (p, p_tf32)


def test_x1_pretrained_full_frame_tile_process_vs_cudnn_fp32(net_pretrained, cuda_device):
    """1008x756 -> 1008x756, tile 510 / pad 10 (run_sr.py --test_tile 510 with the 1x config)."""
    net, sd = net_pretrained
    g = torch.Generator().manual_seed(32)
    x = (torch.rand(1, 3, 756, 1008, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 756, 1008, generator=g).to(cuda_device)
    ref32, ref_tf32 = _fp32_and_tf32(lambda: sftnet.tile_process(sd, x, c, 510, 10, scale=1))
    y = net.tile_process(x, c, 510, 10)
    assert y.shape == (1, 3, 756, 1008) and y.device.type == 'cpu'
    p, p_tf32 = pipeline.psnr(y, ref32), pipeline.psnr(ref_tf32, ref32)
    print(f'x1 1008x756 tile_process(510), pretrained weights: k4nerf vs cuDNN fp32 {p:.2f} dB; cuDNN TF32 vs fp32 {p_tf32:.2f} dB')
    assert p >= 65.0, (p, p_tf32)


# ------------------------------------------------------------------------------------------------
# row windows: every layer computes only the rows inside the remaining receptive field of the kept block
# ------------------------------------------------------------------------------------------------
def test_x1_forward_roi_block_is_bit_identical_to_the_full_forward(net, cuda_device):
    g = torch.Generator().manual_seed(41)
    h, w = 210, 44
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, h, w, generator=g).to(cuda_device)
    full = net(x, c)
    frame = torch.full((3, h + 8, w + 12), -7.0, device=cuda_device)
    for keep in ((0, h, 0, w), (0, 100, 0, w), (101, 131, 3, 40), (180, h, 10, w), (95, 96, 0, 1)):
        y0, y1, x0, x1 = keep
        frame.fill_(-7.0)
        dst = frame[:, 4:4 + (y1 - y0), 8:8 + (x1 - x0)]
        net.forward_roi(x, c, keep, dst)
        assert torch.equal(dst, full[0, :, y0:y1, x0:x1]), keep
        frame[:, 4:4 + (y1 - y0), 8:8 + (x1 - x0)] = -7.0
        assert bool((frame == -7.0).all()), ('wrote outside the destination window', keep)


@pytest.mark.parametrize('world', [2, 3])
def test_x1_row_parts_with_halo_reproduce_the_unsplit_tile(net, cuda_device, world):
    """A tile cut into row parts with receptive_halo() rows of recomputed halo gives bit-identical pixels to the un-split
    tile: the x1 tail (conv_hr + conv_last, 2 LR rows) fits in the trunk's row windows."""
    from k4nerf import dist as kdist
    assert net.receptive_halo() == 80
    g = torch.Generator().manual_seed(21)
    H, W = 300, 40
    x = (torch.rand(1, 3, H, W, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, H, W, generator=g).to(cuda_device)
    ref = net.tile_process(x, c, tile_size=510, tile_pad=10, to_cpu=False)
    assert ref.shape == (1, 3, H, W)
    units = kdist.sr_units(H, W, 510, 10, world, net.receptive_halo())
    assert len(units) == world
    out = torch.zeros_like(ref)
    for u in units:
        sa, sb, xa, xb = u['src']
        assert sb - sa < H
        o = net(x[:, :, sa:sb, xa:xb], c.unsqueeze(0)[:, :, sa:sb, xa:xb])
        ky, kx = u['keep']
        y0, y1, x0, x1 = u['dst']
        out[:, :, y0:y1, x0:x1] = o[:, :, ky:ky + y1 - y0, kx:kx + x1 - x0]
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    full = net.tile_process_sharded(x, c, tile_size=510, tile_pad=10)
    assert torch.equal(full, ref)


def test_x1_forward_roi_extra_destinations_receive_the_same_block(net, cuda_device):
    g = torch.Generator().manual_seed(43)
    h, w = 96, 52
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, h, w, generator=g).to(cuda_device)
    full = net(x, c)
    frames = [torch.full((3, h, w), -7.0, device=cuda_device) for _ in range(3)]
    for keep in ((0, h, 0, w), (10, 61, 3, 40)):
        y0, y1, x0, x1 = keep
        for f in frames:
            f.fill_(-7.0)
        win = lambda f: f[:, y0:y1, x0:x1]
        dst = win(frames[0])
        off = 4 * dst.storage_offset()
        net.forward_roi(x, c, keep, dst, extra=[f.data_ptr() + off for f in frames[1:]])
        for f in frames:
            assert torch.equal(win(f), full[0, :, y0:y1, x0:x1]), keep
            chk = f.clone()
            win(chk).fill_(-7.0)
            assert bool((chk == -7.0).all()), ('wrote outside the destination window', keep)


def test_render_frame_4k_with_a_x1_decoder(cuda_device):
    """The device-resident chain with the 1x config's decoder: a [3, H, W] frame equal to render_viewpoints_sr +
    tile_process + clamp."""
    dev = cuda_device
    st = make_state('cfgA', res=32, regime='fog')
    m = model_from_state(st, dev)
    n = k4nerf.SFTNet(3, 1, 64, 5, 32, 1)
    n.load_state_dict(x1_state_dict(seed=3, scale=1.0))
    n = n.to(dev)
    H, W = 20, 28
    K, c2w = scenes.blender_camera(H, W)
    kw = dict(scenes.RENDER_KW_DVGO)
    sr, lr = render.render_frame_4k(m, n, H, W, K, c2w, False, kw, test_tile=16)
    assert sr.shape == (3, H, W) and sr.is_cuda and float(sr.min()) >= 0 and float(sr.max()) <= 1
    _, depths, _, _, _, feats = render.render_viewpoints_sr(m, np.array([c2w.numpy()]), np.array([[H, W]]), np.array([K]), False, kw)
    x = torch.from_numpy(feats[0]).movedim(-1, 0).unsqueeze(0).to(dev)
    cond = torch.from_numpy(depths[0]).movedim(-1, 0).to(dev)
    ref = n.tile_process(x, cond, tile_size=16).squeeze(0).clamp(0, 1)
    assert ref.shape == (3, H, W)
    assert (sr.cpu() - ref).abs().max().item() < 2e-3
    u8, _ = render.render_frame_4k(m, n, H, W, K, c2w, False, kw, test_tile=16, out_u8=True)
    assert u8.dtype == torch.uint8 and u8.shape == (H, W, 3)
    assert (u8.cpu().float() - (ref * 255).floor().permute(1, 2, 0)).abs().max().item() <= 1


# ------------------------------------------------------------------------------------------------
# C ABI: the scale in k4_srnet_desc, the parameter count, the workspace
# ------------------------------------------------------------------------------------------------
def _create(params, scale, n_params=None):
    keep = [t.detach().float().contiguous() for t in params]
    arr = (C.c_void_p * len(keep))(*[t.data_ptr() for t in keep])
    d = _lib.SrnetDesc()
    d.n_in_colors, d.scale, d.num_feat, d.num_block, d.num_grow_ch, d.num_cond = 3, scale, 64, 5, 32, 1
    d.n_params = len(keep) if n_params is None else n_params
    d.h_params = C.cast(arr, C.POINTER(C.c_void_p))
    out = C.c_void_p()
    st = _lib.lib.k4_srnet_create(C.byref(d), C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(out))
    torch.cuda.synchronize()
    return st, out


def _params(n):
    return [t for cv in n._ordered_convs() for t in (cv.weight, cv.bias)]


def test_x1_capi_scale_and_parameter_count(net, cuda_device):
    p1 = _params(net)
    assert len(p1) == 454
    n4 = k4nerf.SFTNet(3, 4, 64, 5, 32, 1).to(cuda_device)
    p4 = _params(n4)
    assert len(p4) == 458
    st, out = _create(p4, 1)                        # scale 1 with the x4 parameter count
    assert st == K4_ERR_INVALID_ARG and not out.value
    st, out = _create(p1, 4)                        # and the other way round
    assert st == K4_ERR_INVALID_ARG and not out.value
    for s in (2, 3, 8, 0):
        for p in (p1, p4):
            st, out = _create(p, s)
            assert st == K4_ERR_UNSUPPORTED and not out.value, s


def test_x1_capi_forward_workspace_contract(net, cuda_device):
    g = torch.Generator().manual_seed(51)
    h, w = 37, 29
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, h, w, generator=g).to(cuda_device)
    want = net(x, c)
    st, h1 = _create(_params(net), 1)
    assert st == 0 and h1.value
    n4 = k4nerf.SFTNet(3, 4, 64, 5, 32, 1).to(cuda_device)
    st, h4 = _create(_params(n4), 4)
    assert st == 0 and h4.value
    try:
        ws1 = int(_lib.lib.k4_srnet_workspace_bytes(h1, h, w))
        ws4 = int(_lib.lib.k4_srnet_workspace_bytes(h4, h, w))
        assert 0 < ws1 < ws4, (ws1, ws4)
        assert int(_lib.lib.k4_srnet_workspace_bytes(None, h, w)) == ws4
        ws = torch.empty(ws1, dtype=torch.uint8, device=cuda_device)
        out = torch.full((3, h, w), -7.0, device=cuda_device)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        st = _lib.lib.k4_srnet_forward(h1, x.data_ptr(), c.data_ptr(), h, w, out.data_ptr(), ws.data_ptr(), ws1, stream)
        torch.cuda.synchronize()
        assert st == 0
        assert torch.equal(out, want[0])
        st = _lib.lib.k4_srnet_forward(h1, x.data_ptr(), c.data_ptr(), h, w, out.data_ptr(), ws.data_ptr(), ws1 - 1, stream)
        assert st == K4_ERR_WORKSPACE
    finally:
        _lib.lib.k4_srnet_destroy(h1)
        _lib.lib.k4_srnet_destroy(h4)
        torch.cuda.synchronize()


_X4_SCRIPT = r'''
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


def test_x4_after_x1_in_one_process_matches_a_fresh_x4_process(net, cuda_device, tmp_path):
    """No launcher or descriptor state that depends on the tail layout is shared between a x1 and a x4 net: a x4 net
    built and run after x1 nets in this process decodes bit for bit what it decodes in a fresh interpreter."""
    g = torch.Generator().manual_seed(61)
    x = (torch.rand(1, 3, 45, 70, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 45, 70, generator=g).to(cuda_device)
    y1 = net.tile_process(x, c, 32, 10)
    assert y1.shape == (1, 3, 45, 70)
    n4 = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    n4.load_state_dict(sftnet.random_state_dict(seed=3))
    n4 = n4.to(cuda_device)
    here = n4.tile_process(x, c, 32, 10)
    assert torch.equal(net.tile_process(x, c, 32, 10), y1)           # and the x1 net is unchanged by the x4 one
    out = str(tmp_path / 'x4.pt')
    code = _X4_SCRIPT.format(root=ROOT, pkg=os.path.join(ROOT, '4k-nerf_b200'), out=out)
    subprocess.run([sys.executable, '-c', code], check=True, timeout=600)
    fresh = torch.load(out, map_location='cpu', weights_only=False)
    assert here.shape == fresh.shape == (1, 3, 180, 280)
    assert torch.equal(here, fresh)
