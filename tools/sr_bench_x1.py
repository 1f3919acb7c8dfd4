"""x1 VC-Decoder timing beside x4: SFTNet(3, 1, ...) of the 1x configurations (refinement at the input resolution) and
SFTNet(3, 4, ...) (the 4K upsampler), both tile_process(510) on 1008x756, timed in alternating rounds in one process,
then the whole frame of each: march 1008x756 (FOG scene of bench.py) + decode, render_frame_4k.

    python tools/sr_bench_x1.py [--rounds R] [--iters N]

One JSON line per measurement, each with the card's name and power limit read in the same run.  TFLOP/s use the
multiply-accumulates of the layer shapes (macs_per_lr_pixel) times the padded-tile pixel count of sftnet.tile_plan."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
import k4nerf  # noqa: E402
from k4nerf import render  # noqa: E402
from oracle import scenes, sftnet  # noqa: E402
from test_sftnet_x1 import x1_state_dict  # noqa: E402

HLR, WLR = 756, 1008
TILE, PAD = 510, 10


def macs_per_lr_pixel(scale, num_block=5, nf=64, ng=32):
    """Multiply-accumulates per LR pixel of SFTNet(3, scale, nf, num_block, ng, 1), from its layer shapes: a conv of
    cin -> cout with a k x k kernel costs cin * cout * k^2 per pixel of its own grid; conv_up1's grid has 4 pixels per
    LR pixel, the grid of conv_up2 / conv_hr / conv_last scale^2, every other layer's 1."""
    conv = lambda cin, cout, k=3: cin * cout * k * k
    sft = lambda nout: 2 * (conv(ng, ng, 1) + conv(ng, nout, 1))
    condnet = conv(1, 64) + conv(64, 64, 1) + conv(64, 64, 1) + conv(64, 32, 1)
    rdb = sum(conv(nf + c * ng, ng) for c in range(4)) + conv(nf + 4 * ng, nf) + sft(nf) + sft(ng)
    body = conv(3, nf) + condnet + num_block * (3 * rdb + sft(nf)) + sft(nf) + conv(nf, nf)
    tail = conv(nf, nf) * scale ** 2 + conv(nf, 3) * scale ** 2              # conv_hr + conv_last at the output grid
    if scale == 4:
        tail += conv(nf, nf) * 2 ** 2 + conv(nf, nf) * 4 ** 2               # conv_up1 (2x grid), conv_up2 (4x grid)
    return body + tail


def card():
    info = {'card': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info['power_limit'], info['max_sm_clock'] = [s.strip() for s in q.split(',')]
    except Exception as e:          # noqa: BLE001 -- the numbers are still printed, marked as missing the limit
        info['power_limit'] = f'unavailable ({e!r})'
    return info


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'sr_bench_x1 measures the GPU; there is no CPU fallback'
    assert macs_per_lr_pixel(4) == 5188864 and macs_per_lr_pixel(1) == 3872704
    dev = torch.device('cuda', 0)
    hw = card()
    nets = {}
    for s in (4, 1):
        n = k4nerf.SFTNet(3, s, 64, 5, 32, 1)
        n.load_state_dict(sftnet.random_state_dict(seed=3, scale=1.0) if s == 4 else x1_state_dict(seed=3, scale=1.0))
        nets[s] = n.to(dev)
    g = torch.Generator().manual_seed(1)
    img = torch.rand(1, 3, HLR, WLR, generator=g).to(dev)
    cond = torch.rand(1, HLR, WLR, generator=g).to(dev)
    padded = sum((p[1] - p[0]) * (p[3] - p[2]) for p in sftnet.tile_plan(HLR, WLR, TILE, PAD))
    for s in (4, 1):                                   # warm every shape of the timed window
        for _ in range(3):
            nets[s].tile_process(img, cond, TILE, PAD, to_cpu=False)
    torch.cuda.synchronize()
    ms = {4: [], 1: []}
    for _ in range(args.rounds):                       # alternate: both see the same clocks and neighbours
        for s in (4, 1):
            ms[s].append(timed(lambda: nets[s].tile_process(img, cond, TILE, PAD, to_cpu=False), args.iters))
    dec = {}
    for s in (4, 1):
        med = statistics.median(ms[s])
        dec[s] = med
        flop = 2 * macs_per_lr_pixel(s) * padded
        print(json.dumps({'what': f'SFTNet x{s} tile_process({TILE}) 1008x756 -> {s * WLR}x{s * HLR}', 'ms_per_frame': med,
                          'ms_min': min(ms[s]), 'ms_max': max(ms[s]), 'rounds': args.rounds, 'iters': args.iters,
                          'macs_per_lr_pixel': macs_per_lr_pixel(s), 'padded_lr_pixels': padded,
                          'tflops': flop / med / 1e9, **hw}), flush=True)
    print(json.dumps({'what': 'x1 / x4 decode time', 'ratio': dec[1] / dec[4],
                      'mac_ratio': macs_per_lr_pixel(1) / macs_per_lr_pixel(4), **hw}), flush=True)

    # the whole frame: march 1008x756 FOG + decode (render_frame_4k), per scale
    from helpers import make_state, model_from_state
    model = model_from_state(make_state('cfgA', res=160, regime='fog'), dev)
    kw = dict(near=2.0, far=6.0, bg=1, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False)
    K, c2w = scenes.blender_camera(HLR, WLR, theta=30.0, phi=-30.0)
    frame = {s: (lambda s=s: render.render_frame_4k(model, nets[s], HLR, WLR, K, c2w, False, kw, test_tile=TILE)) for s in (4, 1)}
    for s in (4, 1):
        for _ in range(3):
            frame[s]()
    torch.cuda.synchronize()
    fr = {4: [], 1: []}
    for _ in range(args.rounds):
        for s in (4, 1):
            fr[s].append(timed(frame[s], max(1, args.iters // 2)))
    sr, _ = frame[1]()
    assert tuple(sr.shape) == (3, HLR, WLR)
    for s in (4, 1):
        print(json.dumps({'what': f'whole frame x{s}: march 1008x756 FOG + x{s} decode (render_frame_4k, tile {TILE})',
                          'ms_per_frame': statistics.median(fr[s]), 'ms_min': min(fr[s]), 'ms_max': max(fr[s]), **hw}),
              flush=True)


if __name__ == '__main__':
    main()
