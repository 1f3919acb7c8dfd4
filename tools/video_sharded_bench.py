"""Frames per second of run_sr.py --render_video on 1, 2, 4 and 8 GPUs of one node: render.render_video_4k_sharded (frame
i on rank i % world, the round's u8 frames gathered to rank 0) against the single-GPU render.render_video_4k, on the
synthetic cfgA 160^3 fog scene with a x4 decoder, 1008 x 756 LR frames decoded to 4032 x 3024 at test_tile 510.

Each rank count runs as its own torch.distributed.run job (world sizes above the GPU count are skipped).  A job times,
after a warm-up video of one frame per rank:
  sharded      render_video_4k_sharded of --frames frames, the SR frames copied to rank 0's pageable host memory
  no_host_sr   the same with an on_frame that drops the SR frames: the difference is rank 0's 36.6 MB device-to-host
               copy per SR frame, which is the expected limit at many ranks
and the one-rank job also times render_video_4k itself.  Host clock around the whole call, ending with the arrays on
the host.  Prints one JSON line with the card's name and power limit.

    python tools/video_sharded_bench.py [--frames 24] [--ranks 1,2,4,8] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, '4k-nerf_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

H, W = 756, 1008


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else 'unknown'


def worker(frames):
    import numpy as np
    import torch
    import torch.distributed as dist
    import k4nerf
    from k4nerf import render
    from helpers import make_state, model_from_state
    from oracle import scenes, sftnet
    local = int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    dist.init_process_group('nccl', device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    m = model_from_state(make_state('cfgA', res=160, regime='fog'), dev)
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    net.load_state_dict(sftnet.random_state_dict(seed=3, scale=1.0))
    net = net.to(dev)
    kw = dict(scenes.RENDER_KW_DVGO)
    poses, Ks = [], []
    for i in range(frames):
        K, c2w = scenes.blender_camera(H, W, theta=360.0 * i / frames)
        poses.append(c2w.numpy()); Ks.append(K)
    poses, Ks, HW = np.array(poses), np.array(Ks), np.array([[H, W]] * frames)
    args = (m, net, poses, HW, Ks, False, kw)

    def timed(fn):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dist.barrier()
        return time.perf_counter() - t0
    render.render_video_4k_sharded(m, net, poses[:world], HW[:world], Ks[:world], False, kw)          # warm-up
    res = {'ranks': world}
    t = timed(lambda: render.render_video_4k_sharded(*args))
    res['sharded_fps'] = frames / t
    t = timed(lambda: render.render_video_4k_sharded(*args, on_frame=lambda i, sr, lr: None))
    res['no_host_sr_fps'] = frames / t
    if world == 1:
        render.render_video_4k(*args[:2], poses[:1], HW[:1], Ks[:1], False, kw)
        t = timed(lambda: render.render_video_4k(*args))
        res['render_video_4k_fps'] = frames / t
    if rank == 0:
        print('RESULT ' + json.dumps(res), flush=True)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=24)
    ap.add_argument('--ranks', default='1,2,4,8')
    ap.add_argument('--out')
    ap.add_argument('--worker', action='store_true')
    a = ap.parse_args()
    if a.worker:
        return worker(a.frames)
    import socket
    import torch
    n_gpus = torch.cuda.device_count()
    result = {'card': card(), 'n_gpus': n_gpus, 'frames': a.frames, 'lr': [H, W], 'sr': [4 * H, 4 * W], 'runs': []}
    for r in (int(x) for x in a.ranks.split(',')):
        if r > n_gpus:
            result['runs'].append({'ranks': r, 'skipped': f'{n_gpus} GPU(s)'})
            continue
        with socket.socket() as s:
            s.bind(('127.0.0.1', 0))
            port = s.getsockname()[1]
        cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(r), '--master-addr',
               '127.0.0.1', '--master-port', str(port), os.path.abspath(__file__), '--worker', '--frames', str(a.frames)]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
        lines = [l[7:] for l in out.stdout.splitlines() if l.startswith('RESULT ')]
        result['runs'].append(json.loads(lines[-1]) if lines else {'ranks': r, 'error': out.stderr[-2000:]})
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
