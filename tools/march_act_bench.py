"""Frame time of the LLFF MPI model with each rgbnet activation: DirectMPIGO [384,384,256], rgbnet 15-64-64-3 (ws config
6), act_type relu / gauss / lkrelu, one 4032x3024 frame per launch on the warp-specialised wgmma marcher ('ws'), FOG and
SHELL regimes.  The three activations alternate inside every round (7 rounds by default); each timing is CUDA events
around `--reps` back-to-back launches after a warm-up.  Prints one JSON line with per-case medians and ranges (ms per
frame) and the card's name and power limit, read in the same run.

    python tools/march_act_bench.py [--rounds 7] [--reps 3] [--hw 3024 4032] [--xy 384] [--depth 256] [--out FILE]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import torch  # noqa: E402

from helpers import make_state, model_from_state  # noqa: E402
from mpi_act import mpi_model, scale_state_rgbnet  # noqa: E402
from oracle import scenes  # noqa: E402

ACTS = ('relu', 'gauss', 'lkrelu')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--hw', type=int, nargs=2, default=[3024, 4032])
    ap.add_argument('--xy', type=int, default=384)
    ap.add_argument('--depth', type=int, default=256)
    ap.add_argument('--regimes', nargs='+', default=['fog', 'shell'])
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'march_act_bench measures the GPU kernels: no GPU found'
    dev = torch.device('cuda', 0)
    H, W = a.hw
    ro, rd, vd = [t.to(dev) for t in scenes.llff_rays(H, W)]
    kw = dict(scenes.RENDER_KW_MPI)
    kw['render_depth'] = True
    res = {'workload': f'DirectMPIGO [{a.xy},{a.xy},{a.depth}] rgbnet 15-64-64-3, {W}x{H} per launch, mode ws',
           'card': card(), 'rounds': a.rounds, 'reps': a.reps, 'cases': {}}
    for regime in a.regimes:
        st = make_state('cfgB', xy=a.xy, depth=a.depth, regime=regime)
        models = {}
        for act in ACTS:
            s = dict(st)
            s['rgbnet'] = copy.deepcopy(st['rgbnet'])
            if act == 'gauss':
                scale_state_rgbnet(s, act)          # an rgbnet whose Gaussian is not saturated (tests/mpi_act.py)
            models[act] = (model_from_state(s, dev) if act == 'relu' else mpi_model(s, act, dev))
            assert models[act].resolve_mlp_mode('auto') == 'ws'
        del st
        times = {act: [] for act in ACTS}
        for act, m in models.items():             # warm-up: module load, scene build, first launch
            m.render_rays(ro, rd, vd, kw, image_hw=(H, W), mlp_mode='ws')
        torch.cuda.synchronize()
        for r in range(a.rounds):
            for act in (ACTS if r % 2 == 0 else ACTS[::-1]):
                m = models[act]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    m.render_rays(ro, rd, vd, kw, image_hw=(H, W), mlp_mode='ws')
                e1.record()
                torch.cuda.synchronize()
                times[act].append(e0.elapsed_time(e1) / a.reps)
        for act in ACTS:
            t = times[act]
            res['cases'][f'{regime}-{act}'] = {'median_ms': round(statistics.median(t), 3), 'min_ms': round(min(t), 3),
                                               'max_ms': round(max(t), 3)}
        base = statistics.median(times['relu'])
        for act in ACTS[1:]:
            res['cases'][f'{regime}-{act}']['vs_relu'] = round(statistics.median(times[act]) / base, 4)
        del models
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
