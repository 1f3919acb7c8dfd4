#!/usr/bin/env python
"""Where the warp-specialised 4K marcher's cycles go: the bench.py workload (same scene, poses and 4032x3024 frame) run
through the profiled instantiation of k4_march_ws_kernel (k4_testing_march_phases, include/k4nerf.h).

    python tools/march_phases.py [--poses 5] [--regime fog] [--json OUT.json]

Prints, per warpgroup role (marchers, MLP groups), each phase's share of the role's elapsed SM cycles summed over all
CTAs and poses, and the kernel's SM-cycles per shaded sample: the CTAs' elapsed cycles (the longest warpgroup of each)
summed, over the shaded samples.  The profiled kernel reads the SM clock at every phase boundary, so it runs a little
slower than the production kernel; the shares, not its time, are the result.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))

import torch  # noqa: E402


def profile_frame(model, rays, kw, hw, max_ctas=1024):
    """One profiled launch: (phases int64 [n_ctas, 4, K4_PHASE_SLOTS] on the host, counters, render outputs)."""
    from k4nerf import _lib
    dev = rays[0].device
    ph = torch.zeros((max_ctas, 4, _lib.K4_PHASE_SLOTS), dtype=torch.int64, device=dev)
    ret = model.render_rays(*rays, kw, image_hw=hw, mlp_mode='ws', debug=True, phases=ph)
    torch.cuda.synchronize()
    return ph[:ret['n_ctas']].cpu(), ret['counters'].cpu(), ret


def summarise(phases, counters):
    """phases [n, 4, SLOTS] (any number of CTAs of any number of launches), counters = summed k4 debug counters."""
    from k4nerf import _lib
    p = phases.to(torch.float64)
    out = {}
    for role, wgs, names in (('marchers', [0, 1], _lib.MARCHER_PHASES), ('mlp', [2, 3], _lib.MLP_PHASES)):
        sel = p[:, wgs, :]
        elapsed = sel[..., 0].sum().item()
        out[role] = {'elapsed_cycles': elapsed,
                     'share': {nm: sel[..., s].sum().item() / elapsed for s, nm in names.items()},
                     'batches': int(sel[..., _lib.K4_PHASE_SLOTS - 1].sum().item())}
    cta_cycles = p[..., 0].max(dim=1).values.sum().item()
    out['shaded_samples'] = int(counters[2])
    out['batches_counter'] = int(counters[3])
    out['cycles_per_shaded_sample'] = cta_cycles / max(int(counters[2]), 1)
    return out


def print_table(s):
    print(f"{'role':10s} {'phase':12s} {'share':>7s}")
    for role in ('marchers', 'mlp'):
        for nm, v in s[role]['share'].items():
            print(f'{role:10s} {nm:12s} {100 * v:6.1f}%')
        print(f"{role:10s} {'batches':12s} {s[role]['batches']:>7d}")
    print(f"SM-cycles per shaded sample: {s['cycles_per_shaded_sample']:.2f}  "
          f"(shaded samples {s['shaded_samples']}, batches {s['batches_counter']})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--poses', type=int, default=5, help='how many of bench.py\'s poses to profile')
    ap.add_argument('--regime', default='fog', choices=['fog', 'shell'])
    ap.add_argument('--json', default=None, help='also write the summary here')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('march_phases.py: no CUDA device')
    import bench
    import k4nerf
    from oracle import scenes
    dev = torch.device('cuda', 0)
    st, model_from_state = bench.build_scene(args.regime)
    model = model_from_state(st, dev)
    kw = dict(near=2.0, far=6.0, bg=1, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)
    H, W = bench.H4K, bench.W4K
    all_ph, counters = [], torch.zeros(4, dtype=torch.int64)
    for pose in bench.POSES[:args.poses]:
        K, c2w = scenes.blender_camera(H, W, theta=pose[0], phi=pose[1])
        ro, rd, vd = k4nerf.get_rays_of_a_view(H, W, K, c2w, False, False, False, False, device=dev)
        rays = (ro.view(-1, 3), rd.view(-1, 3), vd.view(-1, 3))
        model.render_rays(*rays, kw, image_hw=(H, W), mlp_mode='ws')           # warm-up
        ph, c, _ = profile_frame(model, rays, kw, (H, W))
        all_ph.append(ph)
        counters += c
    s = summarise(torch.cat(all_ph), counters)
    s['gpu'] = torch.cuda.get_device_name(dev)
    print_table(s)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(s, f, indent=1)


if __name__ == '__main__':
    main()
