"""CPU: the x1 VC-Decoder, SFTNet(3, 1, 64, 5, 32, 1) of the reference's 1x configurations (no upsampling; conv_hr and
conv_last run at the input resolution).  The oracle against the reference module's golden vectors
(tests/golden/make_golden_x1.py), the module's parameter names and C-ABI order, its receptive halo, and the sharded
decode at scale 1."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import k4nerf
from oracle import sftnet
from helpers import PRETRAINED_SR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _load(name):
    return torch.load(os.path.join(GOLD, name), map_location='cpu', weights_only=False)


def _sftnet_inputs():
    g = torch.Generator().manual_seed(11)
    x = torch.rand(1, 3, 20, 28, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, 20, 28, generator=g)
    xt = torch.rand(1, 3, 24, 40, generator=g) * 1.2 - 0.1
    ct = torch.rand(1, 24, 40, generator=g)
    return x, c, xt, ct


def x1_state_dict(seed=3, scale=0.5):
    """Seeded x1 parameters: oracle.sftnet.random_state_dict's x4 set without conv_up1 / conv_up2, which a x1 net does
    not register (lib/sr_esrnet.py:430-433).  ``scale`` is the weights' standard-deviation factor."""
    return {k: v for k, v in sftnet.random_state_dict(seed=seed, scale=scale).items()
            if not k.startswith(('conv_up1.', 'conv_up2.'))}


def pretrained_x1_state_dict():
    """run_sr.py:662-663 at scale 1: the seeded x1 parameters with RealESRNet_x4plus.pth loaded on top, strict=False
    (conv_up1 / conv_up2 of the checkpoint have no place in a x1 net).  None where the checkpoint is absent."""
    if not os.path.exists(PRETRAINED_SR):
        return None
    sd = x1_state_dict(seed=3)
    ck = torch.load(PRETRAINED_SR, map_location='cpu', weights_only=False)
    ck = ck['params_ema'] if 'params_ema' in ck else ck['params']
    for k, v in ck.items():
        k = k[7:] if k.startswith('module.') else k
        if k in sd and sd[k].shape == v.shape:
            sd[k] = v.float().clone()
    return sd


def test_x1_oracle_matches_reference_module_output():
    """sftnet_x1_ref.pt was produced by the REFERENCE's lib/sr_esrnet.py SFTNet(scale=1): pins oracle.sftnet at x1."""
    gold = _load('sftnet_x1_ref.pt')
    sd = x1_state_dict(seed=gold['param_seed'])
    x, c, xt, ct = _sftnet_inputs()
    y = sftnet.sftnet_forward(sd, x, c, scale=1)
    assert y.shape == gold['forward'].shape == (1, 3, 20, 28)
    assert (y - gold['forward']).abs().max().item() <= 2e-5
    yt = sftnet.tile_process(sd, xt, ct, tile_size=16, tile_pad=10, scale=1)
    assert yt.shape == gold['tile_process'].shape == (1, 3, 24, 40)
    assert (yt - gold['tile_process']).abs().max().item() <= 2e-5


def test_x1_oracle_with_pretrained_weights_matches_reference_module():
    sd = pretrained_x1_state_dict()
    if sd is None:
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing')
    gold = _load('sftnet_x1_pretrained_ref.pt')
    g = torch.Generator().manual_seed(gold['input_seed'])
    x = torch.rand(1, 3, 40, 48, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, 40, 48, generator=g)
    y = sftnet.sftnet_forward(sd, x, c, scale=1)
    assert y.shape == gold['forward'].shape == (1, 3, 40, 48)
    assert (y - gold['forward']).abs().max().item() <= 2e-5


def test_x1_state_dict_matches_reference_module_and_abi_order():
    gold = _load('sftnet_x1_ref.pt')
    n = k4nerf.SFTNet(3, 1, 64, 5, 32, 1)
    shapes = {k: tuple(v.shape) for k, v in n.state_dict().items()}
    assert shapes == gold['state_dict_shapes']
    assert shapes == {k: tuple(v.shape) for k, v in x1_state_dict(seed=3).items()}
    assert not hasattr(n, 'conv_up1') and not hasattr(n, 'conv_up2')
    convs = n._ordered_convs()
    assert len(convs) == 227                         # 2 * 227 = n_params of include/k4nerf.h at x1, 5 blocks
    assert convs[-3:] == [n.conv_body, n.conv_hr, n.conv_last]
    assert len({id(c) for c in convs}) == 227
    n.load_state_dict(x1_state_dict(seed=3), strict=True)


def test_x1_receptive_halo_and_other_scales():
    assert k4nerf.SFTNet(3, 1, 64, 5, 32, 1).receptive_halo() == 80        # conv_hr + conv_last: 2 LR rows
    assert k4nerf.SFTNet(3, 4, 64, 5, 32, 1).receptive_halo() == 80
    assert k4nerf.SFTNet(3, 1, 64, 2, 32, 1).receptive_halo() == 34
    for s in (2, 3, 8):
        with pytest.raises(NotImplementedError, match='SFTNet\\(3, 1'):
            k4nerf.SFTNet(3, s, 64, 5, 32, 1)


def test_x1_load_network_drops_the_upsampling_convs():
    """run_sr.py:663 on a x1 net: load_network(RealESRNet_x4plus.pth, strict=False) loads conv_first, the RRDB convs,
    conv_body, conv_hr and conv_last; conv_up1.* / conv_up2.* are unexpected keys and dropped."""
    if not os.path.exists(PRETRAINED_SR):
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing')
    n = k4nerf.SFTNet(3, 1, 64, 5, 32, 1)
    n.load_state_dict(x1_state_dict(seed=3))
    n.load_network(PRETRAINED_SR, 'cpu', strict=False)
    want = pretrained_x1_state_dict()
    got = n.state_dict()
    assert set(got) == set(want)
    assert all(torch.equal(got[k], want[k]) for k in want)
    ck = torch.load(PRETRAINED_SR, map_location='cpu', weights_only=False)
    ck = ck['params_ema'] if 'params_ema' in ck else ck['params']
    assert torch.equal(got['conv_hr.weight'], ck['conv_hr.weight'].float())
    assert torch.equal(got['conv_last.weight'], ck['conv_last.weight'].float())


# ---------------------------------------------------------------------------------------------
# decoder sharding at scale 1 (k4nerf.dist.sr_decode_sharded): a stand-in decoder, gloo world 2
# ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fake_decoder_x1(x, c):
    """Stand-in x1 'decoder' with a 2-pixel receptive radius and zero padding (5x5 box filter of img + cond)."""
    import torch.nn.functional as F
    k = torch.ones(3, 1, 5, 5, dtype=x.dtype) / 25
    return F.conv2d(x + c, k, padding=2, groups=3)


def _tile_process_local_x1(fn, img, cond, tile, pad):
    import math
    _, C, H, W = img.shape
    out = img.new_zeros((1, C, H, W))
    c4 = cond.unsqueeze(0)
    for ty in range(math.ceil(H / tile)):
        for tx in range(math.ceil(W / tile)):
            x0, y0 = tx * tile, ty * tile
            x1, y1 = min(x0 + tile, W), min(y0 + tile, H)
            x0p, x1p, y0p, y1p = max(x0 - pad, 0), min(x1 + pad, W), max(y0 - pad, 0), min(y1 + pad, H)
            o = fn(img[:, :, y0p:y1p, x0p:x1p], c4[:, :, y0p:y1p, x0p:x1p])
            out[:, :, y0:y1, x0:x1] = o[:, :, y0 - y0p:y1 - y0p, x0 - x0p:x1 - x0p]
    return out


def _sr_worker_x1(rank, world, port, H, W, tile, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, '4k-nerf_b200'))
    from k4nerf import dist as kdist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    g = torch.Generator().manual_seed(9)
    img = torch.randn(1, 3, H, W, generator=g)
    cond = torch.randn(1, H, W, generator=g)
    ref = _tile_process_local_x1(_fake_decoder_x1, img, cond, tile, 1)
    full = kdist.sr_decode_sharded(_fake_decoder_x1, img, cond, tile, tile_pad=1, scale=1, halo=2)
    q.put((rank, tuple(full.shape) == (1, 3, H, W) and bool(torch.equal(full, ref))))
    dist.destroy_process_group()


@pytest.mark.parametrize('H,W,tile', [(23, 31, 16), (40, 12, 64)])
def test_x1_decoder_sharding_world2_gloo(H, W, tile):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sr_worker_x1, args=(r, 2, port, H, W, tile, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res), res
