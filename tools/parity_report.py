"""Parity report on the GPU box: PSNR / max-abs of every MLP mode against the CPU oracle and, when
oracle/_ref exists, against the reference pipeline on the reference's own kernels.
    python tools/parity_report.py > parity.jsonl"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
from oracle import ops, pipeline  # noqa: E402
from helpers import compare, make_state, model_from_state, rays_for  # noqa: E402


def main():
    dev = torch.device('cuda', 0)
    modes = sys.argv[1:] or ['fp32', 'f16x3', 'f16', 'ws']
    cases = [('cfgA', dict(res=96, regime='fog'), (96, 128)), ('cfgA', dict(res=96, regime='shell'), (96, 128)),
             ('cfgB', dict(xy=96, depth=64, regime='fog'), (72, 96)), ('cfgB', dict(xy=96, depth=64, regime='shell'), (72, 96))]
    have_ref = os.path.exists(ops.ref_ext_path())
    ref_ops = ops.RefExtOps() if have_ref else None
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, kw, hw in cases:
        st = make_state(name, **kw)
        (ro, rd, vd), rkw = rays_for(st, *hw)
        n = ro.shape[0]
        stats = {}
        ref_cpu = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, **rkw)
        ref_gpu = None
        if have_ref:
            ref_gpu = pipeline.forward(pipeline.state_to(st, dev), ro.to(dev), rd.to(dev), vd.to(dev), ref_ops, **rkw)
            c = compare(ref_gpu, ref_cpu, n)
            print(json.dumps({'case': name, **kw, 'pair': 'reference-kernels-pipeline(GPU) vs oracle(CPU)', **c}), flush=True)
        m = model_from_state(st, dev)
        for mode in modes:
            try:
                out = m.render_rays(ro.to(dev), rd.to(dev), vd.to(dev), rkw, image_hw=hw, mlp_mode=mode, debug=True)
            except Exception as e:      # mode not built for this shape
                print(json.dumps({'case': name, **kw, 'mode': mode, 'error': str(e)}), flush=True)
                continue
            c = compare(out, ref_cpu, n)
            cnt = out['counters'].cpu().tolist()
            rec = {'case': name, **kw, 'mode': mode, 'pair': 'k4 vs oracle(CPU)', **c,
                   'S_c_k4': cnt[2], 'S_c_oracle': stats['S_c'], 'S_m_k4': cnt[0], 'S_m_oracle': stats['S_m']}
            print(json.dumps(rec), flush=True)
            if ref_gpu is not None:
                c = compare(out, ref_gpu, n)
                print(json.dumps({'case': name, **kw, 'mode': mode, 'pair': 'k4 vs reference-kernels-pipeline(GPU)', **c}), flush=True)


if __name__ == '__main__':
    main()
