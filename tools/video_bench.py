"""Time of run_sr.py --render_video's three streams: render.render_video_4k against the reference-structured host path,
on a synthetic DVGO scene with a x4 decoder, 1008 x 756 LR frames decoded to 4032 x 3024.

  device   render_video_4k: per frame render_frame_4k, the SR and LR frames quantised on the device, the SR frame copied
           to the host as uint8; the depth video from the device-resident depths at the end.
  host     run_sr.py:1399-1463's structure: render_viewpoints_sr (every frame to the host), tile_process per frame
           with its fp32 result copied to the host, np.array of the SR frames, numpy to8b of both videos, and the depth
           video in numpy (np.percentile and the rainbow table).
Per-frame time: a host clock around the whole call (ending in the data on the host) over --frames frames, after a
one-frame warm-up of each path, divided by --frames.  Peak host memory: each path runs in a child process of its own,
which samples its resident set every 5 ms during the call and reports the peak over the resident set before it.
  kernels  k4_op_masked_quantiles and k4_op_depth_video_u8 alone on --depth-frames random 1008 x 756 depth / bgmap
           frames (CUDA events, median of --reps calls after 3), next to the numpy depth video of the same frames (once).
Prints one JSON line with the card's name, power limit and maximum SM clock read in the same run.

    python tools/video_bench.py [--frames 4] [--depth-frames 120] [--reps 20] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H, W = 756, 1008


def rss_mb():
    with open('/proc/self/statm') as f:
        return int(f.read().split()[1]) * os.sysconf('SC_PAGE_SIZE') / 2 ** 20


class PeakRss(threading.Thread):
    """The largest resident set seen while running, sampled every 5 ms."""

    def __init__(self):
        super().__init__(daemon=True)
        self.peak, self.done = rss_mb(), threading.Event()

    def run(self):
        while not self.done.wait(0.005):
            self.peak = max(self.peak, rss_mb())

    def stop(self):
        self.done.set()
        self.join()
        return max(self.peak, rss_mb())


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def scene(n, dev):
    import k4nerf
    from helpers import make_state, model_from_state
    from oracle import scenes, sftnet
    m = model_from_state(make_state('cfgA', res=160, regime='fog'), dev)
    poses, Ks = [], []
    for i in range(n):
        K, c2w = scenes.blender_camera(H, W, theta=30.0 + 360.0 * i / max(n, 1))
        poses.append(c2w.numpy()); Ks.append(K)
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    net.load_state_dict(sftnet.random_state_dict(seed=3))
    return m, net.to(dev), np.array(poses), np.array([[H, W]] * n), np.array(Ks), dict(scenes.RENDER_KW_DVGO)


def host_path(m, net, poses, HW, Ks, kw, dev):
    """run_sr.py:1399-1463 without the writers (num_cond 1, --test_tile 510)."""
    from k4nerf import render
    from k4nerf.utils import rainbow_lut_u8, to8b
    rgbs, depths, bgmaps, _, _, rgb_features = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw)
    rgbsr = []
    for idx, rgbsave in enumerate(rgb_features):
        rgbtest = torch.from_numpy(rgbsave).movedim(-1, 0).unsqueeze(0).to(dev)
        input_cond = torch.from_numpy(depths).movedim(-1, 1)[idx, :, :, :].to(dev)
        rgb_srtest = net.tile_process(rgbtest, input_cond, tile_size=510).to('cpu')
        rgbsr.append(rgb_srtest.squeeze().movedim(0, -1).detach().clamp(0, 1).numpy())
    rgbsr = np.array(rgbsr)
    sr8, lr8 = to8b(rgbsr), to8b(rgbs)
    return sr8, lr8, numpy_depth_video(depths, bgmaps, rainbow_lut_u8())


def numpy_depth_video(depths, bgmaps, lut):
    depths_vis = depths * (1 - bgmaps) + bgmaps
    dmin, dmax = np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95])
    with np.errstate(divide='ignore', invalid='ignore'):
        x = 1 - np.clip((depths_vis - dmin) / (dmax - dmin), 0, 1)
        xa = x * 256
        xa[xa == 256] = 255
        bad = np.isnan(xa)
        idx = xa.astype(int)
    idx[bad] = 0
    out = lut[idx[..., 0] if idx.ndim == 4 else idx]
    out[bad[..., 0] if bad.ndim == 4 else bad] = 0
    return out


def child(path, n):
    dev = torch.device('cuda', 0)
    from k4nerf import render
    m, net, poses, HW, Ks, kw = scene(n, dev)
    run = (lambda p, h, k: render.render_video_4k(m, net, p, h, k, False, kw, test_tile=510)) if path == 'device' else \
          (lambda p, h, k: host_path(m, net, p, h, k, kw, dev))
    run(poses[:1], HW[:1], Ks[:1])                                      # warm-up: modules, workspaces
    torch.cuda.synchronize()
    base = rss_mb()
    mon = PeakRss()
    mon.start()
    t0 = time.perf_counter()
    out = run(poses, HW, Ks)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = mon.stop()
    print(json.dumps({'path': path, 'frames': n, 'ms_per_frame': 1e3 * dt / n, 'host_mb_before': base,
                      'peak_host_mb_over_before': peak - base, 'shapes': [list(a.shape) for a in out]}), flush=True)


def kernels(nf, reps):
    from k4nerf import _lib
    from k4nerf.utils import _quantile_fractions, rainbow_lut_u8
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(0)
    d = 2 + torch.randn(nf, H, W, generator=g, device=dev)
    b = torch.rand(nf, H, W, generator=g, device=dev) * 0.15
    st = (C.c_int64 * 3)(*d.stride())
    ws = torch.empty(_lib.lib.k4_op_masked_quantiles_workspace_bytes(nf, H, W), dtype=torch.uint8, device=dev)
    res = torch.empty(3, dtype=torch.int64, device=dev)
    out = torch.empty(nf, H, W, 3, dtype=torch.uint8, device=dev)
    q = (C.c_double * 2)(*_quantile_fractions((5, 95)).tolist())
    lut = np.ascontiguousarray(rainbow_lut_u8())
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    quant = lambda: _lib.lib.k4_op_masked_quantiles(C.c_void_p(d.data_ptr()), C.c_void_p(b.data_ptr()), nf, H, W, st, st, q,
                                                    C.c_void_p(res.data_ptr()), C.c_void_p(res.data_ptr() + 16),
                                                    C.c_void_p(ws.data_ptr()), ws.numel(), s)
    cmap = lambda: _lib.lib.k4_op_depth_video_u8(C.c_void_p(d.data_ptr()), C.c_void_p(b.data_ptr()), nf, H, W, st, st,
                                                 C.c_void_p(res.data_ptr()), lut.ctypes.data_as(C.POINTER(C.c_uint8)), 0, 0,
                                                 C.c_void_p(out.data_ptr()), s)
    result = {}
    for name, fn in (('quantiles', quant), ('colormap', cmap)):
        ts = []
        for i in range(reps + 3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            assert fn() == 0
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                ts.append(e0.elapsed_time(e1))
        result[name + '_ms'] = statistics.median(ts)
        result[name + '_ms_range'] = [min(ts), max(ts)]
    n = nf * H * W
    result['quantiles_GB_s'] = 3 * 8 * n / result['quantiles_ms'] / 1e6          # three passes over depth + bgmap
    result['colormap_GB_s'] = (8 + 3) * n / result['colormap_ms'] / 1e6
    t0 = time.perf_counter()
    numpy_depth_video(d.cpu().numpy(), b.cpu().numpy(), lut)
    result['numpy_depth_video_ms'] = 1e3 * (time.perf_counter() - t0)
    result['depth_frames'] = nf
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=4)
    ap.add_argument('--depth-frames', type=int, default=120)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    ap.add_argument('--child', choices=['device', 'host'], default=None)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.frames)
        return
    res = {'card': card(), 'lr': [W, H], 'sr': [4 * W, 4 * H], 'frames': a.frames}
    for path in ('device', 'host'):
        r = subprocess.run([sys.executable, *(['-s'] if sys.flags.no_user_site else []), os.path.abspath(__file__),
                            '--child', path, '--frames', str(a.frames)], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f'{path} path failed:\n{r.stderr[-3000:]}')
        res[path] = json.loads(r.stdout.strip().splitlines()[-1])
    res['speedup_per_frame'] = res['host']['ms_per_frame'] / res['device']['ms_per_frame']
    res['kernels'] = kernels(a.depth_frames, a.reps)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
