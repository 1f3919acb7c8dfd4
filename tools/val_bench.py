"""run_sr.py's joint-stage validation of one view (run_sr.py:1088-1146) on one card: the reference-structured host
block against render.render_val_4k, alternated in one process.

Scene: bench.py's seeded cfgA grid (res 160, SHELL regime), one 1008 x 756 view decoded x4 to 4032 x 3024 by the seeded
decoder (num_cond 1, --test_tile 510), load_sr 1, a seeded [3, H, W]-planar ground truth viewed as [H, W, 3] as
run_sr.py:765-769 builds it, seeded LPIPS-VGG weights (the lpips package is absent).
  host    render_viewpoints_sr, tile_process to the CPU, clamp + .cpu(), numpy MSE, the numpy SSIM, cv2.resize (or the
          numpy restatement without cv2) and rgb_lpips of the resized arrays, both PNGs through the host writer
  device  render.render_val_4k with the same arguments
Each arm is timed with a host clock around one call ending in a device synchronise, --reps times, alternating, after one
warm-up call of each.  The LR report and the per-view lines are printed by both arms and swallowed here.  Prints the
card's name, power limit and max SM clock, then one JSON line (medians and the per-arm samples in seconds).

    python tools/val_bench.py [--reps 3]
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H, W, GRID_RES = 756, 1008, 160


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def host_block(m, net, poses, HW, Ks, kw, gt, srgt, weights, dev, savedir, step=5, sel_b=0):
    """run_sr.py:1088-1146 for load_sr == 1, line for line."""
    from k4nerf import render, utils
    from k4nerf.sr_esrnet import sft_condition
    try:
        from cv2 import resize
    except ImportError:
        resize = lambda x, dsize, fx, fy: utils._resize_quarter_np(x)
    rgbs, depths, bgmaps, psnrs, viewdirs, rgb_features = render.render_viewpoints_sr(
        m, poses, HW, Ks, False, kw, gt_imgs=gt, savedir=savedir, global_step=step)
    out = []
    for idx, rgbsave in enumerate(rgb_features):
        rgbtest = torch.from_numpy(rgbsave).movedim(-1, 0).unsqueeze(0).to(dev)
        cond = sft_condition(net.num_cond, torch.from_numpy(depths[idx]).to(dev), viewdirs[idx], H, W)
        rgb_srtest = net.tile_process(rgbtest, cond, tile_size=510)
        render._write_png(os.path.join(savedir, f'test_{step}.png'), utils.to8b(rgbs[idx]))
        rgb_srsave = rgb_srtest.squeeze().movedim(0, -1).detach().clamp(0, 1).cpu().numpy()
        sr_psnr = -10. * np.log10(np.mean(np.square(rgb_srsave - srgt[idx])))
        sr_ssim = utils.rgb_ssim(rgb_srsave, srgt[idx], max_val=1)
        sr_lpips = utils.rgb_lpips(resize(rgb_srsave, dsize=None, fx=1 / 4, fy=1 / 4),
                                   resize(srgt[idx], dsize=None, fx=1 / 4, fy=1 / 4), 'vgg', device=dev, weights=weights)
        render._write_png(os.path.join(savedir, f'testsr_{step}_{sel_b}.png'), utils.to8b(rgb_srsave))
        out.append((sr_psnr, sr_ssim, sr_lpips))
    return out


def cv2_check(x):
    """How many values of cv2.resize(x, fx=fy=1/4) differ from utils.resize_quarter's, at cv2's default thread count and
    at one thread: the host arm's LPIPS equals the device arm's only where cv2 computes the formula it was matched with."""
    from k4nerf import utils
    try:
        import cv2
    except ImportError:
        return {'cv2': None}
    want = utils._resize_quarter_np(x)
    out = {'cv2': cv2.__version__, 'ipp': bool(cv2.ipp.useIPP()), 'cpus': os.cpu_count(), 'threads': cv2.getNumThreads()}
    out['differ_default_threads'] = int(np.count_nonzero(cv2.resize(x, None, fx=1 / 4, fy=1 / 4) != want))
    n = cv2.getNumThreads()
    cv2.setNumThreads(1)
    out['differ_one_thread'] = int(np.count_nonzero(cv2.resize(x, None, fx=1 / 4, fy=1 / 4) != want))
    cv2.setNumThreads(n)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    import k4nerf
    from k4nerf import render
    from helpers import make_state, model_from_state
    from oracle import lpips as lpips_ref, scenes, sftnet
    dev = torch.device('cuda', 0)
    m = model_from_state(make_state('cfgA', res=GRID_RES, regime='shell'), dev)
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    net.load_state_dict(sftnet.random_state_dict(seed=3, scale=1.0))
    net = net.to(dev)
    K, c2w = scenes.blender_camera(H, W, theta=40.0)
    poses, HW, Ks = np.array([c2w.numpy()]), np.array([[H, W]]), np.array([K])
    kw = dict(scenes.RENDER_KW_DVGO)
    g = torch.Generator().manual_seed(0)
    gt = [torch.rand(H, W, 3, generator=g).numpy()]
    srgt = torch.rand(1, 3, 4 * H, 4 * W, generator=g).movedim(1, -1).numpy()
    weights = lpips_ref.random_state_dict('vgg', seed=1)
    arms = {
        'host': lambda d: host_block(m, net, poses, HW, Ks, kw, gt, srgt, weights, dev, d),
        'device': lambda d: [tuple(v[0] for v in render.render_val_4k(m, net, poses, HW, Ks, False, kw, gt, srgt, 1,
                                                                      savedir=d, global_step=5, lpips_weights=weights)[6:])],
    }
    times = {k: [] for k in arms}
    results = {}
    with tempfile.TemporaryDirectory() as d:
        for rep in range(args.reps + 1):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with contextlib.redirect_stdout(io.StringIO()):
                    results[name] = fn(d)
                torch.cuda.synchronize()
                if rep:
                    times[name].append(time.perf_counter() - t0)
    (hp, hs, hl), (dp, ds, dl) = results['host'][0], results['device'][0]
    print(card())
    print(json.dumps(cv2_check(srgt[0])))
    print(json.dumps({'view': f'{W}x{H} -> {4 * W}x{4 * H}', 'reps': args.reps,
                      'median_s': {k: statistics.median(v) for k, v in times.items()}, 'samples_s': times,
                      'same_psnr': bool(hp == dp), 'same_lpips': hl == dl, 'ssim_diff': abs(hs - ds),
                      'sr_psnr': float(dp), 'sr_ssim': ds, 'sr_lpips': dl}))


if __name__ == '__main__':
    main()
