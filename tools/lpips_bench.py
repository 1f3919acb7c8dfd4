"""Time of LPIPS-VGG: utils.rgb_lpips's kernels (k4_lpips_forward, csrc/k4_lpips.cu) against torch's fp32 evaluation of
the same network (oracle/lpips.py's restatement on cuDNN with its default TF32), on a 4032 x 3024 pair (the joint stage's
4K validation frame) and a 1008 x 756 pair (an LR test view), random weights of the real shapes.

Per size, the two are timed alternately in one run: CUDA events around one k4_lpips_forward call on preallocated
buffers, and around one torch evaluation under no_grad.  Each is the median (and range) of --reps calls after --warmup
calls.  TFLOP/s = 2 x the trunk's multiply-accumulates of both images (from the layer shapes, oracle.lpips.macs) over
the median.  Prints one JSON line, with the card's name, power limit and maximum SM clock read in the same run.

    python tools/lpips_bench.py [--reps 10] [--warmup 3] [--sizes 3024x4032,756x1008] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from k4nerf import _lib, utils  # noqa: E402
from oracle import lpips as ol  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(',')]
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:                                    # the timings stand without it
        return {'name': torch.cuda.get_device_name(), 'error': str(e)}


def stats(ts):
    return {'median_ms': statistics.median(ts), 'min_ms': min(ts), 'max_ms': max(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--sizes', default='3024x4032,756x1008')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('lpips_bench needs a CUDA device')
    dev = torch.device('cuda', 0)
    sd = ol.random_state_dict('vgg', seed=0)
    net = utils.LpipsNet('vgg', sd, dev)
    lib = _lib.lib
    stream = torch.cuda.current_stream(dev)
    res = {'card': card(), 'net': 'vgg', 'reps': args.reps, 'warmup': args.warmup, 'sizes': {}}
    for size in args.sizes.split(','):
        H, W = map(int, size.split('x'))
        g = torch.Generator().manual_seed(H + W)
        a = torch.rand(H, W, 3, generator=g).to(dev)
        b = torch.rand(H, W, 3, generator=g).to(dev)
        ws = torch.empty(lib.k4_lpips_workspace_bytes(net.handle, H, W), dtype=torch.uint8, device=dev)
        out = torch.empty((), dtype=torch.float64, device=dev)
        sa, sb = utils._strides3(a), utils._strides3(b)

        def ours():
            _lib.check(lib.k4_lpips_forward(net.handle, C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), sa, sb, H, W,
                                            C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                            C.c_void_p(stream.cuda_stream)), 'k4_lpips_forward')

        def theirs():
            with torch.no_grad():
                return ol.lpips(sd, 'vgg', a.permute(2, 0, 1), b.permute(2, 0, 1), torch.float32)

        times = {'kernels': [], 'torch_fp32_tf32': []}
        for i in range(args.warmup + args.reps):
            for name, fn in (('kernels', ours), ('torch_fp32_tf32', theirs)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[name].append(e0.elapsed_time(e1))
        flop = 2 * 2 * ol.macs('vgg', H, W)
        r = {'tflop': flop / 1e12}
        for name, ts in times.items():
            r[name] = stats(ts)
            r[name]['tflop_per_s'] = flop / (r[name]['median_ms'] * 1e-3) / 1e12
        r['score_kernels'] = out.item()
        r['score_torch_fp32_tf32'] = theirs().item()
        res['sizes'][f'{W}x{H}'] = r
        del ws
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
