"""CPU: the fused training step's C ABI (k4_train_march_args, k4_train_march_*) and the argument checks of
k4nerf.train_fused.render_loss, all before any CUDA call (there is no GPU here)."""
import ctypes as C
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_args_struct_matches_the_header():
    from k4nerf import _lib
    A = _lib.TrainMarchArgs
    assert C.sizeof(A) == 384
    offs = dict(n_rays=8, world_size=16, k0_dim=28, mask_size=32, mpi_depth=44, xyz_min=48, xyz2ijk_shift=84, act_shift=96,
                interval=104, fast_color_thres=108, stepsize=116, max_world_size=124, rgbnet_depth=128, rgbnet_act_param=148,
                w_main=152, w_rgbper=164, d_rays_o=168, d_bkgd=200, d_mask=224, d_rgbnet_weight=240, d_rgbnet_bias=264,
                d_rgb_marched=288, d_loss_terms=312, d_grad_density=320, d_grad_weight=336, d_grad_bias=360)
    for k, v in offs.items():
        assert getattr(A, k).offset == v, k
    text = open(os.path.join(ROOT, 'include', 'k4nerf.h')).read()
    body = re.search(r'typedef struct k4_train_march_args \{(.*?)\} k4_train_march_args;', text, re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    names = re.findall(r'\**\s*([a-z_0-9]+)\s*(?:\[\d\])?\s*[,;]', body)
    assert names == [f[0] for f in A._fields_]


def test_workspace_bytes():
    from k4nerf import _lib
    lib = _lib.lib
    assert lib.k4_train_march_workspace_bytes(0) == 0 and lib.k4_train_march_workspace_bytes(-4) == 0
    assert lib.k4_train_march_workspace_bytes(1) == 16 + 80
    assert lib.k4_train_march_workspace_bytes(4096) == 16 + 80 * 4096


def _valid(buf, **kw):
    from k4nerf import _lib
    a = _lib.TrainMarchArgs()
    b = C.addressof(buf)
    a.kind, a.rgbnet_act, a.n_rays = _lib.K4_KIND_DMPIGO, _lib.K4_ACT_RELU, 64
    a.world_size[:] = [8, 8, 4]
    a.mask_size[:] = [8, 8, 4]
    a.k0_dim, a.mpi_depth = 12, 4
    a.stepsize, a.interval = 1.0, 64.0
    a.rgbnet_depth, a.rgbnet_width, a.viewbase_pe, a.spatial_pe = 3, 32, 2, 2
    a.w_main = 1.0
    for f in ('d_rays_o', 'd_rays_d', 'd_viewdirs', 'd_target', 'd_density', 'd_k0', 'd_mask', 'd_act_shift_grid',
              'd_rgb_marched', 'd_alphainv_last', 'd_loss', 'd_loss_terms', 'd_grad_density', 'd_grad_k0'):
        setattr(a, f, b)
    for i in range(3):
        a.d_rgbnet_weight[i] = a.d_rgbnet_bias[i] = a.d_grad_weight[i] = a.d_grad_bias[i] = b
    for k, v in kw.items():
        if k in ('world_size', 'mask_size'):
            getattr(a, k)[:] = v
        elif k.startswith('d_rgbnet_weight'):
            a.d_rgbnet_weight[int(k[-1])] = v
        else:
            setattr(a, k, v)
    return a


def _both(a, ws, ws_bytes):
    from k4nerf import _lib
    lib = _lib.lib
    g = C.create_string_buffer(16)
    return (lib.k4_train_march_forward(C.byref(a) if a is not None else None, ws, ws_bytes, None),
            lib.k4_train_march_backward(C.byref(a) if a is not None else None, C.addressof(g), ws, ws_bytes, None))


def test_invalid_arguments_without_a_gpu():
    from k4nerf import _lib
    buf = C.create_string_buffer(1 << 12)
    ws = C.create_string_buffer(1 << 14)
    wsa = (C.addressof(ws) + 15) // 16 * 16
    assert _both(None, wsa, 8192) == (-1, -1)
    bad = [dict(n_rays=0), dict(n_rays=-5), dict(kind=7), dict(kind=-1), dict(rgbnet_act=3), dict(world_size=[0, 8, 4]),
           dict(mask_size=[8, -1, 4]), dict(k0_dim=2), dict(rgbnet_width=0), dict(stepsize=0.0), dict(interval=-1.0),
           dict(w_main=-1.0), dict(d_rays_o=None), dict(d_target=None), dict(d_density=None), dict(d_mask=None),
           dict(d_act_shift_grid=None), dict(mpi_depth=1), dict(d_rgbnet_weight1=None),
           dict(kind=_lib.K4_KIND_DVGO, w_distortion=0.01), dict(rgbnet_depth=0),
           # GaussianActivation.a must be finite and > 0 (act_den = 2 a^2 divides)
           dict(rgbnet_act=_lib.K4_ACT_GAUSS, rgbnet_act_param=0.0), dict(rgbnet_act=_lib.K4_ACT_GAUSS, rgbnet_act_param=-0.05),
           dict(rgbnet_act=_lib.K4_ACT_GAUSS, rgbnet_act_param=float('nan')),
           dict(rgbnet_act=_lib.K4_ACT_GAUSS, rgbnet_act_param=float('inf'))]
    for kw in bad:
        assert _both(_valid(buf, **kw), wsa, 8192) == (-1, -1), kw
    lib = _lib.lib
    g = C.create_string_buffer(16)
    a = _valid(buf)
    for f in ('d_rgb_marched', 'd_alphainv_last', 'd_loss', 'd_loss_terms'):
        b = _valid(buf, **{f: None})
        assert lib.k4_train_march_forward(C.byref(b), wsa, 8192, None) == -1, f
    assert lib.k4_train_march_backward(C.byref(a), None, wsa, 8192, None) == -1
    # workspace: NULL or misaligned is INVALID_ARG, too small is K4_ERR_WORKSPACE
    assert _both(a, None, 8192) == (-1, -1)
    assert _both(a, wsa + 4, 8192) == (-1, -1)
    assert _both(a, wsa, 16 + 80 * 64 - 1) == (-4, -4)


def test_unbuilt_shapes_without_a_gpu():
    from k4nerf import _lib
    buf = C.create_string_buffer(1 << 12)
    ws = C.create_string_buffer(1 << 14)
    wsa = (C.addressof(ws) + 15) // 16 * 16
    for kw in (dict(kind=_lib.K4_KIND_DCVGO), dict(rgbnet_depth=2), dict(rgbnet_depth=4), dict(k0_dim=33),
               dict(rgbnet_width=129), dict(viewbase_pe=11), dict(spatial_pe=11),
               dict(kind=_lib.K4_KIND_DVGO, rgbnet_act=_lib.K4_ACT_GAUSS),
               dict(k0_dim=32, viewbase_pe=10, spatial_pe=6),        # MLP input 32 + 39 + 63 = 134 > 128
               dict(world_size=[2048, 1024, 1024])):
        assert _both(_valid(buf, **kw), wsa, 8192) == (-2, -2), kw


def _dvgo(**kw):
    from k4nerf import DirectVoxGO
    args = dict(num_voxels=8 ** 3, num_voxels_base=8 ** 3, alpha_init=1e-2, rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=16,
                viewbase_pe=2)
    args.update(kw)
    return DirectVoxGO([-1, -1, -1], [1, 1, 1], **args)


def _mpi(**kw):
    from k4nerf import DirectMPIGO
    args = dict(num_voxels=8 * 8 * 4, mpi_depth=4, rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=16, viewbase_pe=1)
    args.update(kw)
    return DirectMPIGO([-1, -1, 0], [1, 1, 1], **args)


def test_render_loss_raises_before_any_launch():
    from k4nerf import _lib
    from k4nerf.train_fused import render_loss
    r = torch.zeros(4, 3)
    kw_d = dict(near=0.2, far=6.0, stepsize=0.5, bg=1)
    kw_m = dict(near=0, far=1, stepsize=1.0, bg=0)
    dcvgo = types.SimpleNamespace(_k4_kind=_lib.K4_KIND_DCVGO)
    with pytest.raises(NotImplementedError):
        render_loss(dcvgo, r, r, r, r, 1, kw_d)
    with pytest.raises(NotImplementedError):
        render_loss(_dvgo(rgbnet_depth=4), r, r, r, r, 1, kw_d, loss_weights=dict(distortion=0))
    with pytest.raises(NotImplementedError):
        render_loss(_dvgo(rgbnet_width=256), r, r, r, r, 1, kw_d, loss_weights=dict(distortion=0))
    with pytest.raises(NotImplementedError):
        render_loss(_mpi(rgbnet_dim=33), r, r, r, r, 1, kw_m)
    with pytest.raises(NotImplementedError):
        render_loss(_mpi(), r, r, r, r, 1, kw_m, loss_weights=dict(nearclip=1.0))
    # the distortion loss needs DirectMPIGO's s / n_max: the reference fails with a KeyError on n_max
    with pytest.raises(ValueError, match='distortion'):
        render_loss(_dvgo(), r, r, r, r, 1, kw_d)
    # loss_weights is taken as given: main alone on DirectVoxGO has no distortion term, so the next check is the rays'
    with pytest.raises(ValueError, match='CUDA'):
        render_loss(_dvgo(), r, r, r, r, 1, kw_d, loss_weights=dict(main=1.0))
    with pytest.raises(ValueError, match='unknown loss weight'):
        render_loss(_mpi(), r, r, r, r, 1, kw_m, loss_weights=dict(tv=1.0))
    # inputs that are not CUDA fp32 [N,3]
    with pytest.raises(ValueError, match='CUDA'):
        render_loss(_mpi(), r, r, r, r, 1, kw_m)
    with pytest.raises(ValueError):
        render_loss(_mpi(), torch.zeros(4, 2), r, r, r, 1, kw_m)
    with pytest.raises(ValueError):
        render_loss(_mpi(), r.double(), r, r, r, 1, kw_m)
