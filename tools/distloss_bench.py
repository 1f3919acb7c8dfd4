"""Time of the distortion loss, forward plus backward: k4nerf's flatten_eff_distloss (csrc/k4_distloss.cu) against
train_ref64.flatten_eff_distloss run in fp32 with autograd on the GPU.  That torch restatement stands in for the
third-party torch_efficient_distloss package, which is not installed here; it is not that package's implementation.

Workloads: the sample list (weights, s, ray_id) of a real training forward of DirectMPIGO with the LLFF shape
([384,384,256] grid, 4096 rays = N_rand of configs/llff/llff_default_lg.py), FOG and SHELL regimes; a
DirectContractedVoxGO batch (4096 rays); a synthetic list of about 8M samples.  For the two models the whole training
step (training forward, run_sr.py's composite loss with the distortion term from k4nerf, backward) is timed too, and
the op's share of it reported.  The op's own kernel time per call comes from a torch.profiler pass of its own, after the
timed rounds.  The implementations alternate inside every round; each timing is CUDA events around
`--reps` back-to-back calls after a warm-up.  Prints one JSON line with medians and ranges (ms) and the card's name and
power limit, read in the same run.

    python tools/distloss_bench.py [--rounds 7] [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import torch  # noqa: E402

import train_ref64 as R  # noqa: E402
from helpers import make_state, model_from_state  # noqa: E402
from k4nerf.torch_efficient_distloss import flatten_eff_distloss  # noqa: E402
from oracle import scenes  # noqa: E402

RESTATEMENT = R.flatten_eff_distloss


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def op_fns(w, s, interval, ray_id):
    wl = w.detach().clone().requires_grad_(True)

    def ours():
        torch.autograd.grad(flatten_eff_distloss(wl, s, interval, ray_id), wl)

    def restatement():
        torch.autograd.grad(RESTATEMENT(wl, s, interval, ray_id), wl)
    return {'k4nerf': ours, 'torch_restatement_fp32': restatement}


def kernel_us(fn, reps):
    """Device time of the op's own kernels (dl_*) per call, from torch.profiler: the end-to-end timings above include
    the host's autograd and launch overhead whenever the host is slower than the GPU."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = sum(getattr(e, 'device_time_total', 0) or getattr(e, 'cuda_time_total', 0)
              for e in prof.key_averages() if 'dl_' in e.key and 'kernel' in e.key)
    return tot / reps


def library_distloss(w, m, interval, ray_id):
    return flatten_eff_distloss(w, m, interval, ray_id) if w.is_cuda else RESTATEMENT(w, m, interval, ray_id)


def model_workload(kind, regime, dev, n_rays=4096):
    g = torch.Generator().manual_seed(0)
    if kind == 'mpi':
        st = make_state('cfgB', xy=384, depth=256, regime=regime)
        ro, rd, vd = scenes.llff_rays(756, 1008)
        kw = dict(scenes.RENDER_KW_MPI)
        name = f'DirectMPIGO [384,384,256] {regime}, {n_rays} rays'
    else:
        st = make_state('cfgC', res=160, regime=regime)
        ro, rd, vd = scenes.blender_rays(756, 1008)
        kw = dict(scenes.RENDER_KW_DCVGO)
        name = f'DirectContractedVoxGO 160^3 {regime}, {n_rays} rays'
    sel = torch.randperm(ro.shape[0], generator=g)[:n_rays]
    ro, rd, vd = (t[sel].contiguous().to(dev) for t in (ro, rd, vd))
    target = torch.rand(n_rays, 3, generator=g).to(dev)
    m = model_from_state(st, dev)
    out = m(ro, rd, vd, global_step=1, is_train=True, **kw)
    w, s, rid = out['weights'].detach().contiguous(), out['s'].detach().contiguous(), out['ray_id'].contiguous()

    def step():
        o = m(ro, rd, vd, global_step=1, is_train=True, **kw)
        R.composite_loss(o, target, n_rays, near_thres=0.5 if kind == 'dcvgo' else None).backward()
        m.zero_grad(set_to_none=True)
    return name, w, s, 1 / out['n_max'], rid, step


def synthetic_workload(dev, target=8_000_000):
    g = torch.Generator().manual_seed(1)
    L = torch.randint(1, 257, (target // 100,), generator=g)
    L = L[:int((torch.cumsum(L, 0) < target).sum()) + 1]
    rid = torch.repeat_interleave(torch.arange(L.numel()), L).to(dev)
    w = (torch.rand(rid.numel(), generator=g) * 0.05).to(dev)
    u = torch.rand(rid.numel(), generator=g).to(dev)
    s = u[torch.argsort(rid.double() * 2 + u.double())].contiguous()
    return f'synthetic, {L.numel()} rays of 1..256 samples', w, s, 1 / 128, rid, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'distloss_bench measures the GPU kernels: no GPU found'
    dev = torch.device('cuda', 0)
    R.flatten_eff_distloss = library_distloss          # composite_loss's distortion term, on the device: k4nerf's
    res = {'stand_in': 'torch_restatement_fp32 is tests/train_ref64.flatten_eff_distloss in fp32 with autograd, standing '
                       'in for the torch_efficient_distloss package (not installed)',
           'card': card(), 'rounds': a.rounds, 'reps': a.reps, 'cases': {}}
    builders = [lambda: model_workload('mpi', 'fog', dev), lambda: model_workload('mpi', 'shell', dev),
                lambda: model_workload('dcvgo', 'fog', dev), lambda: synthetic_workload(dev)]
    for build in builders:
        name, w, s, interval, rid, step = build()
        fns = op_fns(w, s, interval, rid)
        if step is not None:
            fns['training_step'] = step
        for fn in fns.values():                          # warm-up
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        keys = list(fns)
        for r in range(a.rounds):
            for k in (keys if r % 2 == 0 else keys[::-1]):
                times[k].append(timed(fns[k], a.reps if k != 'training_step' else max(1, a.reps // 4)))
        case = {'samples': int(w.numel()), 'rays': int(rid.max()) + 1}
        for k, t in times.items():
            case[k] = {'median_ms': round(statistics.median(t), 4), 'min_ms': round(min(t), 4), 'max_ms': round(max(t), 4)}
        case['k4nerf_kernels_us'] = round(kernel_us(fns['k4nerf'], a.reps), 2)
        if step is not None:
            case['k4nerf_share_of_step'] = round(statistics.median(times['k4nerf']) / statistics.median(times['training_step']), 4)
        case['speedup_vs_restatement'] = round(statistics.median(times['torch_restatement_fp32']) /
                                               statistics.median(times['k4nerf']), 2)
        res['cases'][name] = case
        print(name, json.dumps(case), flush=True)
        del fns, w, s, rid, step
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
