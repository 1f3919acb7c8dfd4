"""Developer timing loop (NOT the contract bench -- see bench.py): rays/s of the fused marcher per
regime and MLP mode, CUDA-event timed.  python tools/quick_bench.py [--res 160] [--hw 756 1008]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from helpers import make_state, model_from_state, rays_for  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=160)
    ap.add_argument('--hw', type=int, nargs=2, default=[756, 1008])
    ap.add_argument('--modes', nargs='+', default=['ws'])
    ap.add_argument('--regimes', nargs='+', default=['fog', 'shell'])
    ap.add_argument('--kind', default='cfgA')
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--linear', action='store_true')
    ap.add_argument('--radius', type=float, default=0.0)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)
    H, W = a.hw
    for regime in a.regimes:
        if a.kind == 'cfgA':
            st = make_state('cfgA', res=a.res, regime=regime)
        elif a.kind == 'cfgC':
            st = make_state('cfgC', res=a.res, regime=regime)
        else:
            st = make_state('cfgB', xy=384, depth=256, regime=regime)
        (ro, rd, vd), kw = rays_for(st, H, W, **({'radius': a.radius} if a.radius else {}))
        m = model_from_state(st, dev)
        ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
        for mode in a.modes:
            hw = None if a.linear else (H, W)
            out = m.render_rays(ro, rd, vd, kw, image_hw=hw, mlp_mode=mode, debug=True)
            torch.cuda.synchronize()
            c = out['counters'].cpu().tolist()
            n_it = 1 if mode == 'fp32' else a.iters
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n_it):
                m.render_rays(ro, rd, vd, kw, image_hw=hw, mlp_mode=mode)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n_it
            n = H * W
            print(json.dumps({'kind': a.kind, 'regime': regime, 'mode': mode, 'rays': n, 'ms': round(ms, 3),
                              'Mrays_s': round(n / ms / 1e3, 2), 'S_m': c[0], 'S_d': c[1], 'S_c': c[2],
                              'batches': c[3], 'Gsamples_s': round(c[2] / ms / 1e6, 3),
                              'rgb_mean': out['rgb_marched'].mean().item()}), flush=True)


if __name__ == '__main__':
    main()
