"""CPU: the view-conditioned VC-Decoder, SFTNet(3, 4, 64, 5, 32, num_cond) with num_cond 63 (the view-direction
embedding) and 64 (depth, then the embedding).  The oracle against the reference module's golden vectors
(tests/golden/make_golden_cond.py), the module's parameter names and C-ABI order, ``sft_condition`` against an
independent numpy statement, the argument checks of the Python and C layers, and the sharded decode of a 64-channel
condition."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import k4nerf
from k4nerf import _lib
from k4nerf.sr_esrnet import sft_condition
from oracle import sftnet
from helpers import PRETRAINED_SR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
INVALID_ARG, UNSUPPORTED = -1, -2


def _load(name):
    return torch.load(os.path.join(GOLD, name), map_location='cpu', weights_only=False)


def unit_viewdirs(n, g):
    v = torch.randn(n, 3, generator=g)
    return v / v.norm(dim=-1, keepdim=True)


def frame_condition(num_cond, H, W, seed):
    """A [num_cond, H, W] condition as run_sr.py builds it: seeded unit view directions, and for 64 a depth-like map
    (a slanted plane with a raised block) in front."""
    g = torch.Generator().manual_seed(seed)
    v = unit_viewdirs(H * W, g)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing='ij')
    depth = 2.0 + 1.5 * xx - 0.5 * yy
    depth[H // 4:H // 2, W // 3:2 * W // 3] -= 1.0
    depth = depth + 0.01 * torch.rand(H, W, generator=g)
    return sft_condition(num_cond, depth, v, H, W)


def golden_inputs(num_cond):
    """x [1,3,20,28] with cond [1,num_cond,20,28] for the plain forward; xt [1,3,24,40] with the 3-D cond [num_cond,24,40]
    of tile_process."""
    g = torch.Generator().manual_seed(31)
    x = torch.rand(1, 3, 20, 28, generator=g) * 1.2 - 0.1
    xt = torch.rand(1, 3, 24, 40, generator=g) * 1.2 - 0.1
    return x, frame_condition(num_cond, 20, 28, 32)[None], xt, frame_condition(num_cond, 24, 40, 33)


def pretrained_inputs():
    g = torch.Generator().manual_seed(34)
    x = torch.rand(1, 3, 40, 48, generator=g) * 1.2 - 0.1
    return x, frame_condition(64, 40, 48, 35)[None]


def pretrained_cond64_state_dict():
    """run_sr.py:662-663 for num_cond 64: the seeded parameters with RealESRNet_x4plus.pth loaded on top, strict=False
    (CondNet keeps its seeded weights: the checkpoint has none).  None where the checkpoint is absent."""
    if not os.path.exists(PRETRAINED_SR):
        return None
    sd = sftnet.random_state_dict(seed=3, num_cond=64)
    ck = torch.load(PRETRAINED_SR, map_location='cpu', weights_only=False)
    ck = ck['params_ema'] if 'params_ema' in ck else ck['params']
    for k, v in ck.items():
        k = k[7:] if k.startswith('module.') else k
        if k in sd and sd[k].shape == v.shape:
            sd[k] = v.float().clone()
    return sd


@pytest.mark.parametrize('num_cond', (63, 64))
def test_cond_oracle_matches_reference_module_output(num_cond):
    """sftnet_cond{63,64}_ref.pt come from the REFERENCE's lib/sr_esrnet.py SFTNet(num_cond=...): pins oracle.sftnet and
    the conditions."""
    gold = _load(f'sftnet_cond{num_cond}_ref.pt')
    assert gold['num_cond'] == num_cond
    sd = sftnet.random_state_dict(seed=gold['param_seed'], num_cond=num_cond)
    x, c, xt, ct = golden_inputs(num_cond)
    assert c.shape == (1, num_cond, 20, 28) and ct.shape == (num_cond, 24, 40)
    y = sftnet.sftnet_forward(sd, x, c)
    assert y.shape == gold['forward'].shape == (1, 3, 80, 112)
    assert (y - gold['forward']).abs().max().item() <= 2e-5
    yt = sftnet.tile_process(sd, xt, ct, tile_size=16, tile_pad=10)
    assert yt.shape == gold['tile_process'].shape == (1, 3, 96, 160)
    assert (yt - gold['tile_process']).abs().max().item() <= 2e-5


def test_cond64_oracle_with_pretrained_weights_matches_reference_module():
    sd = pretrained_cond64_state_dict()
    if sd is None:
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing')
    gold = _load('sftnet_cond64_pretrained_ref.pt')
    x, c = pretrained_inputs()
    y = sftnet.sftnet_forward(sd, x, c)
    assert y.shape == gold['forward'].shape == (1, 3, 160, 192)
    assert (y - gold['forward']).abs().max().item() <= 2e-5


@pytest.mark.parametrize('num_cond', (63, 64))
def test_cond_state_dict_matches_reference_module_and_abi_order(num_cond):
    gold = _load(f'sftnet_cond{num_cond}_ref.pt')
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, num_cond)
    assert n.num_cond == num_cond
    shapes = {k: tuple(v.shape) for k, v in n.state_dict().items()}
    assert shapes == gold['state_dict_shapes']
    assert shapes['CondNet.0.weight'] == (64, num_cond, 3, 3)
    n.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=num_cond), strict=True)
    convs = n._ordered_convs()
    assert len(convs) == 229 and len({id(c) for c in convs}) == 229
    assert convs[:5] == [n.conv_first, n.CondNet[0], n.CondNet[2], n.CondNet[4], n.CondNet[6]]


def test_cond_parameter_names_follow_the_abi_order_of_the_depth_decoder():
    """Only CondNet.0's input width depends on num_cond; the order of the k4_srnet_desc parameter list does not."""
    def order(net):
        names = {id(m): k for k, m in net.named_modules()}
        return [names[id(c)] for c in net._ordered_convs()]
    assert order(k4nerf.SFTNet(3, 4, 64, 5, 32, 64)) == order(k4nerf.SFTNet(3, 4, 64, 5, 32, 1))
    assert order(k4nerf.SFTNet(3, 1, 64, 2, 32, 63)) == order(k4nerf.SFTNet(3, 1, 64, 2, 32, 1))


def test_cond_load_network_keeps_condnet():
    """run_sr.py:663 on a 64-channel net: RealESRNet_x4plus.pth has no CondNet, so load_network(strict=False) works
    unchanged and CondNet.0 keeps its [64, 64, 3, 3] weights."""
    if not os.path.exists(PRETRAINED_SR):
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing')
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, 64)
    n.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=64))
    n.load_network(PRETRAINED_SR, 'cpu', strict=False)
    want = pretrained_cond64_state_dict()
    got = n.state_dict()
    assert set(got) == set(want) and all(torch.equal(got[k], want[k]) for k in want)


def _numpy_condition(num_cond, depth, viewdirs, H, W):
    """run_sr.py:895-912 restated in numpy (fp64 trigonometry of the fp32 arguments): channel 3 + 10 a + i holds
    sin(v_a 2^i), channel 33 + 10 a + i cos(v_a 2^i); depth in front for 64."""
    v = viewdirs.reshape(H * W, 3).numpy()
    out = np.zeros((H * W, 63))
    out[:, :3] = v
    for a in range(3):
        for i in range(10):
            arg = (v[:, a] * np.float32(2.0 ** i)).astype(np.float32).astype(np.float64)
            out[:, 3 + 10 * a + i] = np.sin(arg)
            out[:, 33 + 10 * a + i] = np.cos(arg)
    out = out.reshape(H, W, 63).transpose(2, 0, 1)
    if num_cond == 64:
        out = np.concatenate([depth.reshape(1, H, W).numpy().astype(np.float64), out], 0)
    return out


@pytest.mark.parametrize('num_cond', (1, 63, 64))
@pytest.mark.parametrize('shape', ('flat', 'image'))
def test_sft_condition_matches_a_numpy_statement(num_cond, shape):
    H, W = 7, 11
    g = torch.Generator().manual_seed(40 + num_cond)
    v = unit_viewdirs(H * W, g) * 1.0
    depth = torch.rand(H * W, generator=g) * 4
    vin, din = (v, depth) if shape == 'flat' else (v.view(H, W, 3), depth.view(H, W, 1))
    c = sft_condition(num_cond, din, vin, H, W)
    assert c.shape == (num_cond, H, W) and c.dtype == torch.float32 and c.is_contiguous()
    if num_cond == 1:
        assert torch.equal(c, depth.view(1, H, W))
        return
    want = _numpy_condition(num_cond, depth, v, H, W)
    assert np.abs(c.double().numpy() - want).max() <= 2.0 ** -23          # one fp32 rounding of sin / cos, |value| <= 1
    e0 = 1 if num_cond == 64 else 0
    if num_cond == 64:
        assert torch.equal(c[0], depth.view(H, W))
    assert torch.equal(c[e0:e0 + 3], v.T.reshape(3, H, W))                  # the raw direction first


def test_sft_condition_rejects_other_widths():
    v = torch.zeros(6, 3)
    d = torch.zeros(6)
    for nc in (0, 2, 3, 32, 62, 65, 128):
        with pytest.raises(ValueError, match='num_cond'):
            sft_condition(nc, d, v, 2, 3)


def test_cond_receptive_halo_is_unchanged():
    for nc in (1, 5, 63, 64):
        assert k4nerf.SFTNet(3, 4, 64, 5, 32, nc).receptive_halo() == 80
        assert k4nerf.SFTNet(3, 1, 64, 5, 32, nc).receptive_halo() == 80
    assert k4nerf.SFTNet(3, 4, 64, 2, 32, 64).receptive_halo() == 34


def test_sftnet_rejects_num_cond_out_of_range():
    for nc in (0, -1):
        with pytest.raises(ValueError, match='num_cond'):
            k4nerf.SFTNet(3, 4, 64, 5, 32, nc)
    for nc in (65, 128):
        with pytest.raises(NotImplementedError, match='1..64'):
            k4nerf.SFTNet(3, 4, 64, 5, 32, nc)
    assert k4nerf.SFTNet(3, 4, 64, 1, 32, 2).CondNet[0].weight.shape == (64, 2, 3, 3)


def test_tile_process_rejects_a_4d_or_mismatched_condition():
    """The reference unsqueezes tile_process's condition itself (lib/sr_esrnet.py:474), so a 4-D one would be sliced on
    the wrong axes; here it raises before any work, as does a condition of the wrong width."""
    n = k4nerf.SFTNet(3, 4, 64, 1, 32, 63)
    img = torch.zeros(1, 3, 12, 20)
    for bad in (torch.zeros(1, 63, 12, 20), torch.zeros(64, 12, 20), torch.zeros(63, 12, 21), torch.zeros(1, 12, 20)):
        with pytest.raises(ValueError, match='num_cond'):
            n.tile_process(img, bad, 16)
        with pytest.raises(ValueError, match='num_cond'):
            n.tile_process_sharded(img, bad, 16)
    out = torch.zeros(3, 48, 80)
    with pytest.raises(ValueError, match='num_cond'):
        n.run_units([(img, torch.zeros(1, 1, 12, 20), (0, 12, 0, 20), out)])


def test_c_abi_rejects_num_cond_out_of_range_without_a_gpu():
    """k4_srnet_create: num_cond < 1 is K4_ERR_INVALID_ARG, > 64 K4_ERR_UNSUPPORTED; k4_testing_condnet: num_cond outside
    0..64 is K4_ERR_INVALID_ARG with nothing run.  Both before any CUDA call."""
    lib = _lib.lib
    buf = C.create_string_buffer(64)
    n_params = 2 * 229
    params = (C.c_void_p * n_params)(*([C.addressof(buf)] * n_params))
    for nc, want in ((0, INVALID_ARG), (-3, INVALID_ARG), (65, UNSUPPORTED), (1 << 20, UNSUPPORTED)):
        d = _lib.SrnetDesc()
        d.n_in_colors, d.scale, d.num_feat, d.num_block, d.num_grow_ch, d.num_cond = 3, 4, 64, 5, 32, nc
        d.n_params, d.h_params = n_params, C.cast(params, C.POINTER(C.c_void_p))
        out = C.c_void_p(1)
        assert lib.k4_srnet_create(C.byref(d), None, C.byref(out)) == want, nc
        assert out.value is None
    A = _lib.CondnetTestArgs
    assert C.sizeof(A) == 56 and A.kernel.offset == 48 and A.num_cond.offset == 52
    ptrs = (C.c_void_p * 8)(*([C.addressof(buf)] * 8))
    for nc in (-1, 65, 1000):
        a = A()
        a.h_condnet = C.cast(ptrs, C.POINTER(C.c_void_p))
        a.d_cond_in = a.d_cond_out = a.d_cond16 = C.addressof(buf)
        a.H, a.W, a.y_lo, a.y_hi, a.num_cond = 8, 8, 0, 8, nc
        used = C.c_int32(7)
        assert lib.k4_testing_condnet(C.byref(a), C.byref(used), None) == INVALID_ARG, nc
        assert used.value == -1


# ---------------------------------------------------------------------------------------------
# decoder sharding with a 64-channel condition (k4nerf.dist.sr_decode_sharded): a stand-in decoder, gloo world 2
# ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fake_decoder_cond(x, c):
    """Stand-in x4 'decoder' with a 2-pixel receptive radius and zero padding: a 5x5 box sum of img plus a
    channel-weighted sum of the condition (so a lost, moved or reordered channel changes the result), then nearest x4.
    Integer operands keep every sum exact, whatever order a crop's convolution takes."""
    import torch.nn.functional as F
    nc = c.shape[1]
    cw = (c * torch.arange(1, nc + 1, dtype=c.dtype).view(1, nc, 1, 1)).sum(1, keepdim=True)
    k = torch.ones(3, 1, 5, 5, dtype=x.dtype)
    return F.interpolate(F.conv2d(x + cw, k, padding=2, groups=3), scale_factor=4, mode='nearest')


def _tile_process_local(fn, img, cond, tile, pad, s):
    import math
    _, Cc, H, W = img.shape
    out = img.new_zeros((1, Cc, s * H, s * W))
    c4 = cond.unsqueeze(0)
    for ty in range(math.ceil(H / tile)):
        for tx in range(math.ceil(W / tile)):
            x0, y0 = tx * tile, ty * tile
            x1, y1 = min(x0 + tile, W), min(y0 + tile, H)
            x0p, x1p, y0p, y1p = max(x0 - pad, 0), min(x1 + pad, W), max(y0 - pad, 0), min(y1 + pad, H)
            o = fn(img[:, :, y0p:y1p, x0p:x1p], c4[:, :, y0p:y1p, x0p:x1p])
            out[:, :, s * y0:s * y1, s * x0:s * x1] = o[:, :, s * (y0 - y0p):s * (y1 - y0p), s * (x0 - x0p):s * (x1 - x0p)]
    return out


def _sr_worker_cond(rank, world, port, H, W, tile, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, '4k-nerf_b200'))
    from k4nerf import dist as kdist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    g = torch.Generator().manual_seed(9)
    img = torch.randint(-8, 9, (1, 3, H, W), generator=g).float()
    cond = torch.randint(-4, 5, (64, H, W), generator=g).float()
    ref = _tile_process_local(_fake_decoder_cond, img, cond, tile, 1, 4)
    full = kdist.sr_decode_sharded(_fake_decoder_cond, img, cond, tile, tile_pad=1, scale=4, halo=2)
    q.put((rank, tuple(full.shape) == (1, 3, 4 * H, 4 * W) and bool(torch.equal(full, ref))))
    dist.destroy_process_group()


@pytest.mark.parametrize('H,W,tile', [(23, 31, 16), (40, 12, 64)])
def test_cond64_decoder_sharding_world2_gloo(H, W, tile):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sr_worker_cond, args=(r, 2, port, H, W, tile, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res), res
