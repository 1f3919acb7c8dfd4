"""Time of the SSIM metric: utils.rgb_ssim of CUDA tensors (k4_op_rgb_ssim, csrc/k4_metrics.cu) against its numpy path,
at the LR frame size every validation pass scores (1008 x 756) and at the 4K output size (4032 x 3024), fp32 pairs.

GPU, per size, with and without the map:
  call     utils.rgb_ssim end to end from Python (workspace and output allocation, the launch, and for the mean the 8-byte
           read that synchronises), CUDA events around each call;
  kernels  the two kernels alone: CUDA events around one k4_op_rgb_ssim call on preallocated buffers.
Each is the median (and range) of --reps calls after --warmup calls.  The numpy path runs once per size on the host.
The fp64 operations and the bytes are counted from the shapes (the algorithm's, not the tiles' halo overhead):
  per channel  3 products per input pixel, 5 blurred maps x f taps x (Ho x W vertical + Ho x Wo horizontal) FMAs
               (2 operations each) and about 25 operations of the formula per output;
  bytes        both images read once, plus the fp64 map written when it is asked for.
Against the data sheet of the H100 SXM (700 W): 34 TFLOP/s fp64 without the tensor cores, 3.35 TB/s HBM3; the JSON
says which of the two bounds the kernels and how close they come to it.  Prints one JSON line, with the card's name,
power limit and maximum SM clock read in the same run.

    python tools/ssim_bench.py [--reps 30] [--warmup 5] [--sizes 756x1008,3024x4032] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))

import torch  # noqa: E402

from k4nerf import _lib  # noqa: E402
from k4nerf.utils import _ssim_window, rgb_ssim  # noqa: E402

PEAK_FP64 = 34e12
PEAK_HBM = 3.35e12
F = 11


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def counts(H, W, elem_bytes, with_map):
    Ho, Wo = H - F + 1, W - F + 1
    ops = 3 * (3 * H * W + 2 * 5 * F * (Ho * W + Ho * Wo) + 25 * Ho * Wo)
    nbytes = 2 * 3 * H * W * elem_bytes + (8 * 3 * Ho * Wo if with_map else 0)
    return ops, nbytes


def stats(ts):
    return {'median_ms': statistics.median(ts), 'min_ms': min(ts), 'max_ms': max(ts)}


def time_each(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def kernels_fn(a, b, with_map):
    """One k4_op_rgb_ssim call on buffers allocated once."""
    H, W = a.shape[0], a.shape[1]
    dev = a.device
    ws = torch.empty(_lib.lib.k4_op_rgb_ssim_workspace_bytes(H, W, F), dtype=torch.uint8, device=dev)
    mean = torch.empty((), dtype=torch.float64, device=dev)
    m = torch.empty((H - F + 1, W - F + 1, 3), dtype=torch.float64, device=dev) if with_map else None
    st0, st1 = (C.c_int64 * 3)(*a.stride()), (C.c_int64 * 3)(*b.stride())
    win = (C.c_double * F)(*_ssim_window(F, 1.5).tolist())
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    args = (C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), 0, H, W, st0, st1, win, F, 0.01 ** 2, 0.03 ** 2,
            None if m is None else C.c_void_p(m.data_ptr()), C.c_void_p(mean.data_ptr()), C.c_void_p(ws.data_ptr()),
            ws.numel(), stream)

    def fn():
        _lib.check(_lib.lib.k4_op_rgb_ssim(*args), 'k4_op_rgb_ssim')
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--sizes', default='756x1008,3024x4032', help='H x W pairs')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ssim_bench needs a CUDA device')
    assert args.reps >= 20, 'the medians are taken over at least 20 calls'
    dev = torch.device('cuda', 0)
    res = {'device': torch.cuda.get_device_name(dev), 'power_limit_and_max_sm_clock': card(), 'filter_size': F,
           'dtype': 'float32', 'reps': args.reps, 'warmup': args.warmup, 'sizes': {}}
    for s in args.sizes.split(','):
        H, W = (int(v) for v in s.split('x'))
        g = torch.Generator().manual_seed(H + W)
        a = torch.rand(H, W, 3, generator=g)
        b = (a + 0.1 * torch.randn(H, W, 3, generator=g)).clamp(0, 1)
        t0 = time.perf_counter()
        ref = rgb_ssim(a.numpy(), b.numpy(), 1)
        t_np = time.perf_counter() - t0
        ad, bd = a.to(dev), b.to(dev)
        got = rgb_ssim(ad, bd, 1)
        row = {'numpy_s': t_np, 'ssim_gpu': got, 'ssim_numpy': ref, 'abs_diff': abs(got - ref)}
        for with_map in (False, True):
            tag = 'map' if with_map else 'mean'
            call = stats(time_each(lambda: rgb_ssim(ad, bd, 1, return_map=with_map), args.reps, args.warmup))
            kern = stats(time_each(kernels_fn(ad, bd, with_map), args.reps, args.warmup))
            ops, nbytes = counts(H, W, 4, with_map)
            t = kern['median_ms'] * 1e-3
            t_ops, t_bytes = ops / PEAK_FP64, nbytes / PEAK_HBM
            row[tag] = {'call': call, 'kernels': kern, 'fp64_ops': ops, 'bytes': nbytes,
                        'fp64_tflops': ops / t / 1e12, 'hbm_tbps': nbytes / t / 1e12,
                        'bound': 'fp64' if t_ops >= t_bytes else 'hbm', 'share_of_bound': max(t_ops, t_bytes) / t,
                        'speedup_vs_numpy': t_np / (call['median_ms'] * 1e-3)}
        res['sizes'][f'{W}x{H}'] = row
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
