"""Time of one scene-training step: the fused path (k4nerf.train_fused.render_loss + backward, csrc/k4_train_march.cu)
against the materialised one (model(..., is_train=True) + train_ref64.composite_loss + backward, the loss of run_sr.py
with k4nerf's distortion op), on the same model, rays and target.

Workloads: DirectMPIGO [384,384,256] FOG and SHELL with 4096 rays (DESIGN 3.5's; configs/llff/llff_default_lg.py's
N_rand), DirectVoxGO 160^3 with rgbnet 39-128-128-3 FOG and the coarse no-MLP DirectVoxGO 100^3 FOG with 8192 rays
(configs/syn/syn_default.py's fine and coarse stages).  Timed per workload:
  step       forward, loss and backward, gradients set to None before each step;
  step+adam  the same plus the MaskedAdam step (skip_zero_grad), whose dense gradient zeroing and Adam pass over the
             grids are a floor that fusion does not remove.
The two paths alternate inside every round; each timing is CUDA events around --reps back-to-back steps after a warm-up;
medians and ranges in ms.  Kernel times per step come from a separate torch.profiler pass.  Also recorded: the largest
gradient difference between the paths relative to the gradient's largest magnitude, FLOPs and bytes per fused step
computed from the shapes and the sample counts, and the card's name and power limit read in the same run.

    python tools/train_step_bench.py [--rounds 5] [--reps 10] [--out FILE]
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
from k4nerf import MaskedAdam, train_fused  # noqa: E402
from k4nerf._scene import linear_layers  # noqa: E402
from k4nerf.torch_efficient_distloss import flatten_eff_distloss  # noqa: E402
from oracle import pipeline, scenes  # noqa: E402

LW = dict(main=1.0, entropy_last=0.01, distortion=0.01, rgbper=0.1)


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


def dvgo_state(res, rgbnet_dim, width):
    st = pipeline.dvgo_state([-1, -1, -1], [1, 1, 1], num_voxels=res ** 3, num_voxels_base=res ** 3, alpha_init=1e-2,
                             fast_color_thres=1e-4, rgbnet_dim=rgbnet_dim, rgbnet_direct=True, rgbnet_depth=3,
                             rgbnet_width=width, viewbase_pe=4)
    scenes.fill_grids(st, 'fog')
    if rgbnet_dim:
        scenes.fill_rgbnet(st)
    st.update(_num_voxels=res ** 3, _num_voxels_base=res ** 3, _alpha_init=1e-2)
    return st


def workload(name, dev):
    g = torch.Generator().manual_seed(0)
    if name.startswith('mpi'):
        st = make_state('cfgB', xy=384, depth=256, regime=name.split('_')[1])
        ro, rd, vd = scenes.llff_rays(756, 1008)
        kw, n = dict(scenes.RENDER_KW_MPI), 4096
        lw = dict(LW)
    else:
        st = dvgo_state(160, 12, 128) if name == 'dvgo_fine' else dvgo_state(100, 0, 0)
        ro, rd, vd = scenes.blender_rays(756, 1008)
        kw, n = dict(scenes.RENDER_KW_DVGO), 8192
        lw = dict(LW, distortion=0.0)
    sel = torch.randperm(ro.shape[0], generator=g)[:n]
    ro, rd, vd = (t[sel].contiguous().to(dev) for t in (ro, rd, vd))
    target = torch.rand(n, 3, generator=g).to(dev)
    return model_from_state(st, dev), ro, rd, vd, target, kw, lw


def counts(m, ro, rd, vd, kw):
    """samples (occupied / composited / shaded) of one step, from the materialised forward with hooks"""
    cap = {}
    hs = [m.density.register_forward_hook(lambda mod, i, o: cap.__setitem__('occ', o.shape[0])),
          m.k0.register_forward_hook(lambda mod, i, o: cap.__setitem__('shaded', o.shape[0]))]
    m(ro, rd, vd, global_step=1, is_train=True, **kw)
    for h in hs:
        h.remove()
    return cap['occ'], cap['shaded']


def flops_bytes(m, n_rays, occ, shaded):
    """FLOPs and bytes of one fused step from the shapes: the MLP forward twice (forward kernel, re-march) and its
    backward (2x the forward for data and weight gradients); 8-corner gathers of density (+1 channel) per occupied sample
    twice and of k0 per shaded sample twice, the gradients' 8 atomics per channel; rays, targets and per-ray totals."""
    layers = linear_layers(m.rgbnet)
    mlp = sum(2 * l.in_features * l.out_features for l in layers)
    C = m.k0.grid.shape[1]
    flops = shaded * mlp * 4 + (occ * 2 * 16) + shaded * C * 16 * 3
    byts = 2 * occ * 8 * 4 + 2 * shaded * 8 * 4 * C + occ * 8 * 4 + shaded * 8 * 4 * C + n_rays * (12 * 4 + 64 * 2 + 16)
    return int(flops), int(byts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'train_step_bench measures the GPU kernels: no GPU found'
    dev = torch.device('cuda', 0)
    R.flatten_eff_distloss = flatten_eff_distloss           # composite_loss's distortion term: k4nerf's CUDA op
    res = {'card': card(), 'rounds': a.rounds, 'reps': a.reps, 'cases': {}}
    names = {'mpi_fog': 'DirectMPIGO [384,384,256] FOG, 4096 rays', 'mpi_shell': 'DirectMPIGO [384,384,256] SHELL, 4096 rays',
             'dvgo_fine': 'DirectVoxGO 160^3 39-128-128-3 FOG, 8192 rays', 'dvgo_coarse': 'DirectVoxGO 100^3 no MLP FOG, 8192 rays'}
    for key, title in names.items():
        m, ro, rd, vd, target, kw, lw = workload(key, dev)
        n = ro.shape[0]
        opt = MaskedAdam([{'params': [p], 'lr': 1e-3, 'skip_zero_grad': True} for p in m.parameters() if p.requires_grad])

        def fused():
            m.zero_grad(set_to_none=True)
            train_fused.render_loss(m, ro, rd, vd, target, 1, kw, loss_weights=lw)[0].backward()

        def materialised():
            m.zero_grad(set_to_none=True)
            o = m(ro, rd, vd, global_step=1, is_train=True, **kw)
            R.composite_loss(o, target, n, weights=dict(lw, nearclip=0.0)).backward()

        # gradient difference at this size (before any optimiser step)
        fused()
        gf = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
        materialised()
        gm = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
        diff = {k: float((gf[k] - gm[k]).abs().max() / gm[k].abs().max().clamp_min(1e-30)) for k in gm}
        occ, shaded = counts(m, ro, rd, vd, kw)
        del gf, gm
        # timing: parameters stay fixed for the step-only rows; the Adam rows step them (both paths alike)
        fns = {'fused_step': fused, 'materialised_step': materialised,
               'fused_step+adam': lambda: (fused(), opt.step()), 'materialised_step+adam': lambda: (materialised(), opt.step())}
        state = {k: v.clone() for k, v in m.state_dict().items()}
        for fn in fns.values():
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        keys = list(fns)
        for r in range(a.rounds):
            for k in (keys if r % 2 == 0 else keys[::-1]):
                times[k].append(timed(fns[k], a.reps))
        m.load_state_dict(state)
        case = {'rays': n, 'occupied_samples': occ, 'shaded_samples': shaded,
                'max_rel_grad_diff_fused_vs_materialised': diff}
        for k, t in times.items():
            case[k] = {'median_ms': round(statistics.median(t), 3), 'min_ms': round(min(t), 3), 'max_ms': round(max(t), 3)}
        case['speedup_step'] = round(case['materialised_step']['median_ms'] / case['fused_step']['median_ms'], 2)
        case['speedup_step+adam'] = round(case['materialised_step+adam']['median_ms'] / case['fused_step+adam']['median_ms'], 2)
        f, b = flops_bytes(m, n, occ, shaded)
        case['fused_flops'], case['fused_bytes'] = f, b
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                fused()
            torch.cuda.synchronize()
        ka = {e.key: (getattr(e, 'device_time_total', 0) or 0) / a.reps for e in prof.key_averages()}
        case['fused_kernels_us'] = {k.split('(')[0].split('<')[0][-40:]: round(v, 1) for k, v in ka.items() if v > 1.0}
        res['cases'][title] = case
        print(title, json.dumps(case), flush=True)
        del m, opt, fns, state
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
