"""GPU: the VC-Decoder (SFTNet) conv pipeline through the C ABI against (i) golden vectors produced
by the REFERENCE's own lib/sr_esrnet.py (tests/golden/sftnet_ref.pt) and (ii) the functional
oracle.  Convolution operands are fp16 with fp32 accumulation (the reference's cuDNN convs run
with TF32 operands by default), the trunk / SFT / CondNet math is fp32: bar = 60 dB PSNR."""
import os

import pytest
import torch

import k4nerf
from oracle import pipeline, sftnet
from helpers import pretrained_sr_state_dict

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _inputs():
    g = torch.Generator().manual_seed(11)
    x = torch.rand(1, 3, 20, 28, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, 20, 28, generator=g)
    xt = torch.rand(1, 3, 24, 40, generator=g) * 1.2 - 0.1
    ct = torch.rand(1, 24, 40, generator=g)
    return x, c, xt, ct


@pytest.fixture(scope='module')
def net(cuda_device):
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    n.load_state_dict(sftnet.random_state_dict(seed=3))
    return n.to(cuda_device)


def test_forward_matches_reference_golden(net, cuda_device):
    gold = torch.load(os.path.join(GOLD, 'sftnet_ref.pt'), map_location='cpu', weights_only=False)
    x, c, _, _ = _inputs()
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    assert y.shape == gold['forward'].shape
    p = pipeline.psnr(y, gold['forward'])
    print('SFTNet forward PSNR vs reference', p, 'maxabs', (y - gold['forward']).abs().max().item(),
          'ref range', gold['forward'].min().item(), gold['forward'].max().item())
    assert p >= 60.0, p


def test_tile_process_matches_reference_golden(net, cuda_device):
    gold = torch.load(os.path.join(GOLD, 'sftnet_ref.pt'), map_location='cpu', weights_only=False)
    _, _, xt, ct = _inputs()
    y = net.tile_process(xt.to(cuda_device), ct.to(cuda_device), tile_size=16, tile_pad=10)
    assert y.device.type == 'cpu' and y.shape == gold['tile_process'].shape
    p = pipeline.psnr(y, gold['tile_process'])
    assert p >= 60.0, p


@pytest.mark.parametrize('hw', [(19, 13), (8, 8), (33, 50), (1, 7)])
def test_ragged_sizes_match_oracle(net, cuda_device, hw):
    """Sizes that are not multiples of the 16x8 pixel tile, down to a single row."""
    h, w = hw
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1, 3, h, w, generator=g)
    c = torch.rand(1, 1, h, w, generator=g)
    sd = sftnet.random_state_dict(seed=3)
    ref = sftnet.sftnet_forward(sd, x, c)
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    p = pipeline.psnr(y, ref)
    assert p >= 60.0, (hw, p)


def test_parameter_update_rebuilds_device_copy(net, cuda_device):
    x, c, _, _ = _inputs()
    a = net(x.to(cuda_device), c.to(cuda_device)).clone()
    with torch.no_grad():
        net.conv_last.bias.add_(0.25)
    b = net(x.to(cuda_device), c.to(cuda_device))
    assert abs((b - a).mean().item() - 0.25) < 1e-3
    with torch.no_grad():
        net.conv_last.bias.sub_(0.25)


@pytest.mark.parametrize('world', [2, 3])
def test_row_parts_with_halo_reproduce_the_unsplit_tile(net, cuda_device, world):
    """Multi-GPU decoder sharding (k4nerf.dist.sr_units): a tile cut into row parts with
    SFTNet.receptive_halo() rows of recomputed halo gives bit-identical pixels to the un-split
    tile (simulated ranks on one GPU: same units, run one after another)."""
    from k4nerf import dist as kdist
    assert net.receptive_halo() == 80
    g = torch.Generator().manual_seed(21)
    H, W = 300, 40
    x = (torch.rand(1, 3, H, W, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, H, W, generator=g).to(cuda_device)
    ref = net.tile_process(x, c, tile_size=510, tile_pad=10, to_cpu=False)
    units = kdist.sr_units(H, W, 510, 10, world, net.receptive_halo())
    assert len(units) == world
    out = torch.zeros_like(ref)
    for u in units:
        sa, sb, xa, xb = u['src']
        assert sb - sa < H                       # really a part, with a non-clipped halo on one side at least
        o = net(x[:, :, sa:sb, xa:xb], c.unsqueeze(0)[:, :, sa:sb, xa:xb])
        ky, kx = u['keep']
        y0, y1, x0, x1 = u['dst']
        out[:, :, 4 * y0:4 * y1, 4 * x0:4 * x1] = o[:, :, 4 * ky:4 * (ky + y1 - y0), 4 * kx:4 * (kx + x1 - x0)]
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    # and through the collective-free single-process path of the sharded driver
    full = net.tile_process_sharded(x, c, tile_size=510, tile_pad=10)
    assert torch.equal(full, ref)


# ------------------------------------------------------------------------------------------------
# real weights, real sizes (VERDICT r1 "weak" #1): pretrained/RealESRNet_x4plus.pth loaded strict=False as
# run_sr.py:663 does, the reference's largest tile (520x520) and the whole 1008x756 tile_process(510),
# against oracle.sftnet on cuDNN in true fp32 (TF32 off).  Bar: >= 65 dB; the reference's own default
# arithmetic (cuDNN TF32) is measured beside it on the same input for context.
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def net_pretrained(cuda_device):
    sd = pretrained_sr_state_dict()
    if sd is None:
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing (python oracle/build_ref.py where /root/reference exists)')
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    n.load_state_dict(sd)
    return n.to(cuda_device), {k: v.to(cuda_device) for k, v in sd.items()}


def _fp32_and_tf32(fn):
    """fn() evaluated with cuDNN/cuBLAS in true fp32 and in the reference's default TF32 mode."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
        a = fn()
        torch.backends.cudnn.allow_tf32 = True; torch.backends.cuda.matmul.allow_tf32 = True
        b = fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return a, b


def test_pretrained_forward_matches_reference_module_golden(net_pretrained, cuda_device):
    """Golden vector produced by the REFERENCE module with the shipped checkpoint (tests/golden/make_golden.py)."""
    net, _ = net_pretrained
    gold = torch.load(os.path.join(GOLD, 'sftnet_pretrained_ref.pt'), map_location='cpu', weights_only=False)
    g = torch.Generator().manual_seed(12)
    x = torch.rand(1, 3, 40, 48, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, 40, 48, generator=g)
    y = net(x.to(cuda_device), c.to(cuda_device)).cpu()
    p = pipeline.psnr(y, gold['forward'])
    print('pretrained SFTNet vs reference-module golden: PSNR', p, 'maxabs', (y - gold['forward']).abs().max().item())
    assert p >= 65.0, p


def test_pretrained_520_tile_vs_cudnn_fp32(net_pretrained, cuda_device):
    net, sd = net_pretrained
    g = torch.Generator().manual_seed(31)
    x = (torch.rand(1, 3, 520, 520, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, 520, 520, generator=g).to(cuda_device)
    ref32, ref_tf32 = _fp32_and_tf32(lambda: sftnet.sftnet_forward(sd, x, c))
    y = net(x, c)
    p, p_tf32 = pipeline.psnr(y.cpu(), ref32.cpu()), pipeline.psnr(ref_tf32.cpu(), ref32.cpu())
    print(f'520x520 tile, pretrained weights: k4nerf vs cuDNN fp32 {p:.2f} dB (maxabs {(y - ref32).abs().max().item():.3e}); '
          f'cuDNN TF32 (the reference default) vs cuDNN fp32 {p_tf32:.2f} dB')
    assert y.shape == (1, 3, 2080, 2080)
    assert p >= 65.0, (p, p_tf32)


def test_pretrained_full_frame_tile_process_vs_cudnn_fp32(net_pretrained, cuda_device):
    """BASELINE.json configs[3]: 1008x756 -> 4032x3024, tile 510 / pad 10 (run_sr.py --test_tile 510)."""
    net, sd = net_pretrained
    g = torch.Generator().manual_seed(32)
    x = (torch.rand(1, 3, 756, 1008, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 756, 1008, generator=g).to(cuda_device)
    ref32, ref_tf32 = _fp32_and_tf32(lambda: sftnet.tile_process(sd, x, c, 510, 10))
    y = net.tile_process(x, c, 510, 10)
    assert y.shape == (1, 3, 3024, 4032) and y.device.type == 'cpu'
    p, p_tf32 = pipeline.psnr(y, ref32), pipeline.psnr(ref_tf32, ref32)
    print(f'1008x756 tile_process(510), pretrained weights: k4nerf vs cuDNN fp32 {p:.2f} dB; cuDNN TF32 vs fp32 {p_tf32:.2f} dB')
    assert p >= 65.0, (p, p_tf32)


def test_large_magnitude_activations_do_not_overflow_fp16(cuda_device):
    """Conv / SFT operands are fp16: weights scaled so that the trunk reaches ~1e3 and the SFT modulation
    multiplies it further.  Every fp32 -> fp16 conversion of a computed activation or condition in the kernels
    saturates (cvt.rn.satfinite; CondNet's hi + lo split and its fp16 condition included), so no
    inf/nan may appear and the result must stay close to the fp32 network wherever the fp32 network's own
    intermediate values are representable."""
    sd = sftnet.random_state_dict(seed=5, scale=1.0)
    for k in sd:
        if k.startswith('conv_first'):
            sd[k] = sd[k] * 400.0
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    n.load_state_dict(sd)
    n = n.to(cuda_device)
    g = torch.Generator().manual_seed(6)
    x = torch.rand(1, 3, 40, 56, generator=g).to(cuda_device)
    c = torch.rand(1, 1, 40, 56, generator=g).to(cuda_device)
    sdd = {k: v.to(cuda_device) for k, v in sd.items()}
    ref32, _ = _fp32_and_tf32(lambda: sftnet.sftnet_forward(sdd, x, c))
    y = n(x, c)
    assert torch.isfinite(y).all(), 'fp16 overflow in the decoder'
    rel = (y - ref32).abs().max().item() / ref32.abs().max().item()
    print('large-magnitude decoder: ref range', ref32.abs().max().item(), 'rel maxabs', rel)
    assert rel <= 2e-2, rel


def test_forward_roi_block_is_bit_identical_to_the_full_forward(net, cuda_device):
    """k4_srnet_forward_roi: only the rows inside the remaining receptive field of the kept block are computed by every
    layer and the last convolution writes the block straight into a strided destination."""
    g = torch.Generator().manual_seed(41)
    h, w = 210, 44
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, h, w, generator=g).to(cuda_device)
    full = net(x, c)
    frame = torch.full((3, 4 * h + 8, 4 * w + 12), -7.0, device=cuda_device)
    for keep in ((0, h, 0, w), (0, 100, 0, w), (101, 131, 3, 40), (180, h, 10, w), (95, 96, 0, 1)):
        y0, y1, x0, x1 = keep
        frame.fill_(-7.0)
        dst = frame[:, 4:4 + 4 * (y1 - y0), 8:8 + 4 * (x1 - x0)]
        net.forward_roi(x, c, keep, dst)
        assert torch.equal(dst, full[0, :, 4 * y0:4 * y1, 4 * x0:4 * x1]), keep
        frame[:, 4:4 + 4 * (y1 - y0), 8:8 + 4 * (x1 - x0)] = -7.0
        assert bool((frame == -7.0).all()), ('wrote outside the destination window', keep)


def test_tile_process_streams_and_pdl_do_not_change_results(net, cuda_device):
    g = torch.Generator().manual_seed(42)
    x = (torch.rand(1, 3, 150, 170, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 150, 170, generator=g).to(cuda_device)
    a = net.tile_process(x, c, tile_size=64, tile_pad=10, to_cpu=False, streams=1)
    b = net.tile_process(x, c, tile_size=64, tile_pad=10, to_cpu=False, streams=2)
    d = net.tile_process(x, c, tile_size=64, tile_pad=10, to_cpu=False, streams=3)
    assert torch.equal(a, b) and torch.equal(a, d)
    ref = sftnet.tile_process(sftnet.random_state_dict(seed=3), x.cpu(), c.cpu(), 64, 10)
    assert pipeline.psnr(a.cpu(), ref) >= 60.0


def test_fused_sft_epilogues_match_the_separate_sft_passes(net, cuda_device, monkeypatch):
    """Default: every SFT layer runs in the epilogue of the convolution that produces its input (mma.sync on the accumulator
    fragments, csrc/k4_sr.cu epilogue_sft); K4_SR_FUSE_SFT=0: 36 separate SFT passes (sft_mma_kernel) per tile (the round-1
    structure).  Same operands (fp16 weights / activations), different accumulation order: both within the decoder's bar of
    the fp32 network and far closer to each other."""
    g = torch.Generator().manual_seed(77)
    x = (torch.rand(1, 3, 70, 90, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, 70, 90, generator=g).to(cuda_device)
    monkeypatch.delenv('K4_SR_FUSE_SFT', raising=False)
    a = net(x, c).clone()
    monkeypatch.setenv('K4_SR_FUSE_SFT', '0')
    b = net(x, c).clone()
    monkeypatch.delenv('K4_SR_FUSE_SFT', raising=False)
    ref = sftnet.sftnet_forward(sftnet.random_state_dict(seed=3), x.cpu(), c.cpu())
    pa, pb, pab = pipeline.psnr(a.cpu(), ref), pipeline.psnr(b.cpu(), ref), pipeline.psnr(a.cpu(), b.cpu())
    print('fused vs fp32', pa, 'unfused vs fp32', pb, 'fused vs unfused', pab)
    assert pa >= 60.0 and pb >= 60.0 and pab >= 66.0


def test_forward_roi_extra_destinations_receive_the_same_block(net, cuda_device):
    """k4_srnet_forward_roi_peers: the last convolution stores the kept block into further frames too (on a multi-GPU
    node: the other ranks' peer-mapped frames; here: two more local buffers), same window, same strides."""
    g = torch.Generator().manual_seed(43)
    h, w = 96, 52
    x = (torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1).to(cuda_device)
    c = torch.rand(1, 1, h, w, generator=g).to(cuda_device)
    full = net(x, c)
    frames = [torch.full((3, 4 * h, 4 * w), -7.0, device=cuda_device) for _ in range(3)]
    for keep in ((0, h, 0, w), (10, 61, 3, 40)):
        y0, y1, x0, x1 = keep
        for f in frames:
            f.fill_(-7.0)
        win = lambda f: f[:, 4 * y0:4 * y1, 4 * x0:4 * x1]
        dst = win(frames[0])
        off = 4 * dst.storage_offset()
        net.forward_roi(x, c, keep, dst, extra=[f.data_ptr() + off for f in frames[1:]])
        for f in frames:
            assert torch.equal(win(f), full[0, :, 4 * y0:4 * y1, 4 * x0:4 * x1]), keep
            chk = f.clone()
            win(chk).fill_(-7.0)
            assert bool((chk == -7.0).all()), ('wrote outside the destination window', keep)
