"""Cost of the SFT condition's width: SFTNet(3, 4, 64, 5, 32, num_cond) with num_cond 1 (depth), 63 (the view-direction
embedding) and 64 (depth + embedding), tile_process(510) of 1008x756 -> 4032x3024, timed in alternating rounds in one
process; then one torch.profiler run per width for the CondNet kernel's time per tile.

    python tools/sr_bench_cond.py [--rounds R] [--iters N]

One JSON line per measurement, each with the card's name and power limit read in the same run."""
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
from oracle import sftnet  # noqa: E402
from test_sftnet_cond import frame_condition  # noqa: E402

HLR, WLR = 756, 1008
TILE, PAD = 510, 10
WIDTHS = (1, 63, 64)


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
    assert torch.cuda.is_available(), 'sr_bench_cond measures the GPU; there is no CPU fallback'
    dev = torch.device('cuda', 0)
    hw = card()
    g = torch.Generator().manual_seed(1)
    img = torch.rand(1, 3, HLR, WLR, generator=g).to(dev)
    nets, conds = {}, {}
    for nc in WIDTHS:
        n = k4nerf.SFTNet(3, 4, 64, 5, 32, nc)
        n.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=nc, scale=1.0))
        nets[nc] = n.to(dev)
        conds[nc] = (torch.rand(1, HLR, WLR, generator=g) if nc == 1 else frame_condition(nc, HLR, WLR, 2)).to(dev)
    run = {nc: (lambda nc=nc: nets[nc].tile_process(img, conds[nc], TILE, PAD, to_cpu=False)) for nc in WIDTHS}
    for nc in WIDTHS:                                  # warm every shape of the timed window
        for _ in range(3):
            run[nc]()
    torch.cuda.synchronize()
    ms = {nc: [] for nc in WIDTHS}
    for _ in range(args.rounds):                       # alternate: every width sees the same clocks and neighbours
        for nc in WIDTHS:
            ms[nc].append(timed(run[nc], args.iters))
    for nc in WIDTHS:
        print(json.dumps({'what': f'SFTNet x4 num_cond {nc} tile_process({TILE}) 1008x756 -> 4032x3024',
                          'ms_per_frame': statistics.median(ms[nc]), 'ms_min': min(ms[nc]), 'ms_max': max(ms[nc]),
                          'rounds': args.rounds, 'iters': args.iters, **hw}), flush=True)
    base = statistics.median(ms[1])
    print(json.dumps({'what': 'decode time relative to num_cond 1',
                      **{f'num_cond_{nc}': statistics.median(ms[nc]) / base for nc in WIDTHS[1:]}, **hw}), flush=True)

    # the CondNet kernel per tile: one profiled tile_process per width, in a run of its own after the timed rounds
    from torch.profiler import ProfilerActivity, profile
    ntiles = len(sftnet.tile_plan(HLR, WLR, TILE, PAD))
    for nc in WIDTHS:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run[nc]()
            torch.cuda.synchronize()
        tot, count, frame = 0.0, 0, 0.0
        for ev in prof.key_averages():
            t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0.0)
            frame += t
            if 'condnet' in ev.key:
                tot += t
                count += ev.count
        print(json.dumps({'what': f'CondNet kernel, num_cond {nc}', 'us_per_tile': tot / ntiles, 'launches': count,
                          'tiles': ntiles, 'share_of_kernel_time': tot / frame if frame else None, **hw}), flush=True)


if __name__ == '__main__':
    main()
