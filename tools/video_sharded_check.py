"""torchrun check of render_video_4k_sharded: on rank dst its three arrays, and its on_frame calls, equal the single-GPU
render_video_4k's bit for bit, for x4 (num_cond 1 / 64) and x1 decoders, with and without render_video_flipy /
render_video_rot90 and render_factor, for 1, 3 and 5 frames.  Prints one JSON line on rank 0.

  torchrun --nproc-per-node N tools/video_sharded_check.py [--backend nccl|gloo] [--same-gpu]

--same-gpu puts every rank on cuda:0 (with gloo: two processes sharing one GPU exercise the whole path)."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import k4nerf  # noqa: E402
from k4nerf import render  # noqa: E402
from helpers import make_state, model_from_state  # noqa: E402
from oracle import scenes, sftnet  # noqa: E402
from test_sftnet_x1 import x1_state_dict  # noqa: E402

H, W = 20, 28


def main():
    backend = sys.argv[sys.argv.index('--backend') + 1] if '--backend' in sys.argv else 'nccl'
    local = int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', 0 if '--same-gpu' in sys.argv else local)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, **({'device_id': dev} if backend == 'nccl' else {}))
    rank, world = dist.get_rank(), dist.get_world_size()
    # the shell regime leaves bgmap < 0.1 on part of the frame; fp32 MLP: frames reproduce bit for bit
    m = model_from_state(make_state('cfgA', res=32, regime='shell'), dev)
    m.mlp_mode = 'fp32'
    poses, Ks = [], []
    for th in (30.0, 75.0, 120.0, 165.0, 210.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    poses, Ks, HW = np.array(poses), np.array(Ks), np.array([[H, W]] * 5)
    kw = dict(scenes.RENDER_KW_DVGO)

    def net(scale, nc):
        n = k4nerf.SFTNet(3, scale, 64, 5, 32, nc)
        n.load_state_dict(x1_state_dict(seed=3) if scale == 1 else sftnet.random_state_dict(seed=3, num_cond=nc))
        return n.to(dev)
    nets = {'x4c1': net(4, 1), 'x4c64': net(4, 64), 'x1c1': net(1, 1)}
    cases = []
    for name in nets:
        for n in (1, 3, 5):
            cases.append(dict(net=name, n=n, dst=(n % world)))
    cases += [dict(net='x4c1', n=3, dst=0, render_video_flipy=True, render_video_rot90=1),
              dict(net='x4c64', n=5, dst=world - 1, render_video_rot90=2),
              dict(net='x1c1', n=3, dst=0, render_video_flipy=True),
              dict(net='x4c1', n=5, dst=0, render_factor=2),
              dict(net='x4c64', n=5, dst=world - 1, on_frame=True, render_video_rot90=3),
              dict(net='x4c1', n=1, dst=0, on_frame=True)]
    res = {'world': world, 'backend': backend, 'cases': []}
    for c in cases:
        c = dict(c)
        name, n, dst, with_on_frame = c.pop('net'), c.pop('n'), c.pop('dst'), c.pop('on_frame', False)
        args = (m, nets[name], poses[:n], HW[:n], Ks[:n], False, kw)
        want_frames, got_frames = [], []
        rec = lambda seen: (lambda i, sr, lr: seen.append((i, sr.cpu().numpy(), lr.cpu().numpy())))
        want = render.render_video_4k(*args, test_tile=16, on_frame=rec(want_frames) if with_on_frame else None, **c)
        got = render.render_video_4k_sharded(*args, test_tile=16, on_frame=rec(got_frames) if with_on_frame else None,
                                             group=None, dst=dst, **c)
        if rank == dst:
            ok = all((g is None and w is None) or (g is not None and w is not None and np.array_equal(g, w))
                     for g, w in zip(got, want))
            ok = ok and [f[0] for f in got_frames] == [f[0] for f in want_frames]
            ok = ok and all(np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) for a, b in zip(got_frames, want_frames))
        else:
            ok = got == (None, None, None) and got_frames == []
        t = torch.tensor([int(ok)], dtype=torch.int32, device=dev if backend == 'nccl' else 'cpu')
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        res['cases'].append({'net': name, 'n': n, 'dst': dst, 'on_frame': with_on_frame, **c, 'identical': bool(t.item())})
    if rank == 0:
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
