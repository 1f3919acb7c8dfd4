"""PNG encoding of 4032 x 3024 frames: k4_png_encode on the device against the host writers, on one card.

Frames: the SR output of render.render_frame_4k (1008 x 756 marched, x4 decoded, uint8) on bench.py's seeded SHELL and
FOG scenes with the pretrained decoder oracle/_ref/RealESRNet_x4plus.pth (seeded CondNet, strict=False, as
run_sr.py:662-663), a constant frame, a smooth gradient and uniform noise.
  device      k4_png_encode alone: CUDA events around each call, median of --reps calls after 3 warm-up calls
  device+d2h  utils.png_encode: encode, the length read and the bytes copied to the host (host clock), median
  PIL / cv2   Image.save(format='png') and cv2.imencode('.png') with their defaults (host clock, median of --cpu-reps)
Bytes of each writer's file, the ratio to PIL's.  Prints the card's name and power limit, then one JSON line.

    python tools/png_bench.py [--reps 20] [--cpu-reps 3]
"""
import argparse
import ctypes as C
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H, W = 756, 1008
PRETRAINED = os.path.join(ROOT, 'oracle', '_ref', 'RealESRNet_x4plus.pth')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def decoder(dev):
    import k4nerf
    from oracle import sftnet
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    sd = sftnet.random_state_dict(seed=3)
    ck = torch.load(PRETRAINED, map_location='cpu', weights_only=False)
    ck = ck.get('params_ema', ck.get('params', ck))
    sd.update({k: v for k, v in ck.items() if k in sd and sd[k].shape == v.shape})
    net.load_state_dict(sd)
    return net.to(dev)


def frames(dev):
    from k4nerf import render
    from helpers import make_state, model_from_state
    from oracle import scenes
    net = decoder(dev)
    out = {}
    for regime in ('shell', 'fog'):
        m = model_from_state(make_state('cfgA', res=160, regime=regime), dev)
        K, c2w = scenes.blender_camera(H, W, theta=30.0)
        out[f'decoder_{regime}'] = render.render_frame_4k(m, net, H, W, K, c2w.numpy(), False,
                                                          dict(scenes.RENDER_KW_DVGO), out_u8=True)[0]
    yy, xx = torch.meshgrid(torch.arange(3024, device=dev), torch.arange(4032, device=dev), indexing='ij')
    out['constant'] = torch.full((3024, 4032, 3), 128, dtype=torch.uint8, device=dev)
    out['gradient'] = torch.stack([xx * 255 // 4031, yy * 255 // 3023, (xx + yy) * 255 // 7054], -1).to(torch.uint8)
    g = torch.Generator(device=dev).manual_seed(0)
    out['noise'] = torch.randint(0, 256, (3024, 4032, 3), dtype=torch.uint8, device=dev, generator=g)
    return out


def time_device(frame, reps):
    from k4nerf import _lib
    dev = frame.device
    Hf, Wf = frame.shape[:2]
    bound = _lib.lib.k4_png_encode_bound(Hf, Wf)
    ws = torch.empty(_lib.lib.k4_png_workspace_bytes(Hf, Wf), dtype=torch.uint8, device=dev)
    out = torch.empty(bound, dtype=torch.uint8, device=dev)
    n = torch.empty((), dtype=torch.int64, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    args = (C.c_void_p(frame.data_ptr()), Hf, Wf, C.c_void_p(out.data_ptr()), bound, C.c_void_p(n.data_ptr()),
            C.c_void_p(ws.data_ptr()), ws.numel(), stream)
    ts = []
    for i in range(reps + 3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(_lib.lib.k4_png_encode(*args), 'k4_png_encode')
        e1.record()
        e1.synchronize()
        if i >= 3:
            ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def time_host(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--cpu-reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('png_bench needs a CUDA device')
    from PIL import Image
    import cv2
    from k4nerf.utils import png_encode
    c = card()
    print('card:', c, flush=True)
    dev = torch.device('cuda', 0)
    res = {'card': c, 'host_cpus': os.cpu_count(), 'frames': {}}
    for name, f in frames(dev).items():
        host = f.cpu().numpy()
        dev_ms = time_device(f, a.reps)
        png_encode(f)
        d2h_ms, data = time_host(lambda: png_encode(f), a.reps)
        pil_ms, pil_bytes = time_host(lambda: _pil(host), a.cpu_reps)
        cv_ms, cv_bytes = time_host(lambda: cv2.imencode('.png', host[..., ::-1])[1].nbytes, a.cpu_reps)
        r = dict(device_ms=round(dev_ms, 2), device_d2h_ms=round(d2h_ms, 2), pil_ms=round(pil_ms, 1), cv2_ms=round(cv_ms, 1),
                 bytes=len(data), pil_bytes=pil_bytes, cv2_bytes=cv_bytes, ratio_to_pil=round(len(data) / pil_bytes, 4))
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(data)).convert('RGB')), host), name
        res['frames'][name] = r
        print(name, r, flush=True)
    print(json.dumps(res))


def _pil(host):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(host).save(buf, format='png')
    return buf.tell()


if __name__ == '__main__':
    main()
