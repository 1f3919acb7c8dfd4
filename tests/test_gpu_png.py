"""GPU: PNG files encoded on the device (k4_png_encode, csrc/k4_png.cu; utils.png_encode / write_png) -- every chunk's
CRC, the zlib stream and its Adler-32, the filtered stream byte for byte against the numpy restatement, PIL / cv2
decoding the input pixels, at edge shapes, segment boundaries, long matches, the stored fallback and a 4K decoder
frame; and render.render_test_4k against render_viewpoints_sr, render_frame_4k and the LR dumps."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import k4nerf
from k4nerf import _lib, render
from k4nerf.utils import png_encode, to8b, write_png
from helpers import make_state, model_from_state
from oracle import scenes, sftnet
from png_ref import filter_np, read_png

pytestmark = pytest.mark.gpu
SEG = _lib.K4_PNG_SEG


def _decode_pil(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert('RGB'))


def _check(frame, dev, pil=True):
    """Encode ``frame`` (numpy u8 [H, W, 3]) on the device; check the file; return its bytes."""
    data = png_encode(torch.from_numpy(np.ascontiguousarray(frame)).to(dev))
    H, W = frame.shape[:2]
    h, w, stream, types = read_png(data)
    assert (h, w) == (H, W) and types == ['IHDR', 'IDAT', 'IEND']
    assert np.array_equal(stream, filter_np(frame))
    assert len(data) <= _lib.lib.k4_png_encode_bound(H, W)
    if pil:
        assert np.array_equal(_decode_pil(data), frame)
        try:
            import cv2
        except ImportError:
            cv2 = None
        if cv2 is not None:
            got = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)
            assert np.array_equal(got[..., ::-1], frame)
    return data


def _rng(seed):
    return np.random.default_rng(seed)


@pytest.mark.parametrize('H,W', [(1, 1), (1, 7), (1, 1000), (9, 1), (700, 1), (5, 5), (37, 41), (63, 129), (100, 333)])
def test_shapes(cuda_device, H, W):
    g = _rng(H * 1000 + W)
    yy, xx = np.mgrid[0:H, 0:W]
    smooth = np.stack([(xx * 3 + yy) % 256, (xx + 2 * yy) % 256, (xx * yy) % 256], -1)
    _check(np.clip(smooth + g.integers(-2, 3, smooth.shape), 0, 255).astype(np.uint8), cuda_device)


@pytest.mark.parametrize('H,W,nbytes', [(1, 21845, 2 * SEG), (24576, 1, 3 * SEG), (1, 32768, 3 * SEG + 1),
                                         (1, 43690, 4 * SEG - 1), (2, 5461, SEG)])
def test_segment_boundaries(cuda_device, H, W, nbytes):
    """Filtered streams of exactly k segments and k segments +- 1 byte."""
    assert H * (1 + 3 * W) == nbytes
    g = _rng(W)
    f = (np.arange(H * W * 3).reshape(H, W, 3) // 7 % 256).astype(np.uint8)
    f[..., 1] ^= g.integers(0, 4, (H, W), dtype=np.uint8)
    _check(f, cuda_device)


@pytest.mark.parametrize('value', [0, 1, 200])
@pytest.mark.parametrize('H,W', [(1, 70000), (300, 301), (3024, 4032)])
def test_constant_frames(cuda_device, value, H, W):
    """Maximum-length matches at distance 1 and runs across segment boundaries."""
    f = np.full((H, W, 3), value, np.uint8)
    data = _check(f, cuda_device, pil=H * W < 10 ** 6)
    assert len(data) < H * (1 + 3 * W) / 100


def test_matches_at_distance_32768(cuda_device):
    """Rows A, B, A, B, ... of random bytes with 1 + 3 W = 16384: the filtered stream repeats with a period of exactly
    32768 bytes and has no shorter repeat, so the file compresses only through matches at distance 32768."""
    g = _rng(5)
    W = 5461
    a, b = g.integers(0, 256, (2, W, 3), dtype=np.uint8)
    f = np.stack([a if y % 2 == 0 else b for y in range(40)])
    data = _check(f, cuda_device)
    assert len(data) < 0.25 * f.size


@pytest.mark.parametrize('H,W', [(1, 1), (17, 19), (256, 1000), (3024, 4032)])
def test_uniform_noise_takes_stored_blocks(cuda_device, H, W):
    f = _rng(H + W).integers(0, 256, (H, W, 3), dtype=np.uint8)
    data = _check(f, cuda_device, pil=H * W < 10 ** 6)
    assert len(data) <= _lib.lib.k4_png_encode_bound(H, W)


@pytest.fixture(scope='module')
def frame4k(cuda_device):
    """A 4032 x 3024 SR frame: a 1008 x 756 render of a seeded scene through the seeded x4 decoder."""
    m = model_from_state(make_state('cfgA', res=48, regime='shell'), cuda_device)
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    net.load_state_dict(sftnet.random_state_dict(seed=3))
    net = net.to(cuda_device)
    K, c2w = scenes.blender_camera(756, 1008, theta=40.0)
    u8, _ = render.render_frame_4k(m, net, 756, 1008, K, c2w.numpy(), False, dict(scenes.RENDER_KW_DVGO), out_u8=True)
    assert tuple(u8.shape) == (3024, 4032, 3)
    return u8


def test_4k_decoder_frame_round_trip_and_determinism(cuda_device, frame4k):
    f = frame4k.cpu().numpy()
    data = _check(f, cuda_device)
    assert png_encode(frame4k) == data


def test_encode_does_not_synchronise(cuda_device, frame4k):
    H, W = frame4k.shape[:2]
    dev = cuda_device
    bound = _lib.lib.k4_png_encode_bound(H, W)
    ws = torch.empty(_lib.lib.k4_png_workspace_bytes(H, W), dtype=torch.uint8, device=dev)
    out = torch.empty(bound, dtype=torch.uint8, device=dev)
    n = torch.empty((), dtype=torch.int64, device=dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    torch.cuda.set_sync_debug_mode('error')
    try:
        with torch.cuda.stream(side):
            for _ in range(2):
                _lib.check(_lib.lib.k4_png_encode(C.c_void_p(frame4k.data_ptr()), H, W, C.c_void_p(out.data_ptr()), bound,
                                                  C.c_void_p(n.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                  C.c_void_p(side.cuda_stream)))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side.synchronize()
    assert out[:int(n.item())].cpu().numpy().tobytes() == png_encode(frame4k)


def test_write_png_chooses_by_device(cuda_device, tmp_path):
    f = _rng(1).integers(0, 256, (20, 30, 3), dtype=np.uint8)
    write_png(str(tmp_path / 'dev.png'), torch.from_numpy(f).to(cuda_device))
    write_png(str(tmp_path / 'host.png'), f)
    for name in ('dev.png', 'host.png'):
        assert np.array_equal(_decode_pil((tmp_path / name).read_bytes()), f)
    assert (tmp_path / 'dev.png').read_bytes() == png_encode(torch.from_numpy(f).to(cuda_device))
    with pytest.raises(TypeError):
        write_png(str(tmp_path / 'x.png'), [[1, 2, 3]])
    with pytest.raises(ValueError):
        png_encode(torch.zeros(4, 4, 3, device=cuda_device))                    # float32
    with pytest.raises(ValueError):
        png_encode(torch.zeros(4, 4, 4, dtype=torch.uint8, device=cuda_device))  # RGBA


# ---- render_test_4k ---------------------------------------------------------------------------------
H, W, N = 24, 32, 2


@pytest.fixture(scope='module')
def scene(cuda_device):
    m = model_from_state(make_state('cfgA', res=32, regime='shell'), cuda_device)
    m.mlp_mode = 'fp32'                                # sequential per-ray accumulation: frames reproduce bit for bit
    poses, Ks = [], []
    for th in (30.0, 100.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    return m, np.array(poses), np.array([[H, W]] * N), np.array(Ks), dict(scenes.RENDER_KW_DVGO)


@pytest.mark.parametrize('scale,nc', [(4, 1), (4, 64), (1, 1), (1, 64)])
def test_render_test_4k(scene, cuda_device, tmp_path, scale, nc):
    m, poses, HW, Ks, kw = scene
    net = k4nerf.SFTNet(3, scale, 64, 5, 32, nc)
    sd = sftnet.random_state_dict(seed=3, num_cond=nc)
    if scale == 1:                                     # a x1 net has no conv_up1 / conv_up2 (lib/sr_esrnet.py:430-433)
        sd = {k: v for k, v in sd.items() if not k.startswith(('conv_up1.', 'conv_up2.'))}
    net.load_state_dict(sd)
    net = net.to(cuda_device)
    g = torch.Generator().manual_seed(9)
    gt = [torch.rand(H, W, 3, generator=g).numpy() for _ in range(N)]
    want_dir, got_dir = tmp_path / 'want', tmp_path / 'got'
    want_dir.mkdir(); got_dir.mkdir()
    want = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw, gt_imgs=gt, savedir=str(want_dir), dump_images=True,
                                       global_step=7)
    got = render.render_test_4k(m, net, poses, HW, Ks, False, kw, gt_imgs=gt, savedir=str(got_dir), ckpt_name='fine_last',
                                dump_images=True, global_step=7, test_tile=16)
    for i in (0, 1, 2, 5):
        assert got[i].dtype == want[i].dtype and np.array_equal(got[i], want[i]), i
    assert got[3] == want[3]
    assert len(got[4]) == N and all(torch.equal(a, b) for a, b in zip(got[4], want[4]))
    names = sorted(os.listdir(got_dir))
    assert names == sorted([f'e7_{i:03d}.png' for i in range(N)] + [f'fine_last_{i:03d}.png' for i in range(N)])
    for i in range(N):
        lr_want = _decode_pil((want_dir / f'e7_{i:03d}.png').read_bytes())
        assert np.array_equal(lr_want, to8b(want[0][i]))
        assert np.array_equal(_decode_pil((got_dir / f'e7_{i:03d}.png').read_bytes()), lr_want)
        u8, _ = render.render_frame_4k(m, net, H, W, Ks[i], poses[i], False, kw, test_tile=16, out_u8=True)
        assert np.array_equal(_decode_pil((got_dir / f'fine_last_{i:03d}.png').read_bytes()), u8.cpu().numpy())
