"""One scene-training step's render and loss on two fused kernels (csrc/k4_train_march.cu).

``render_loss`` is ``model(rays_o, rays_d, viewdirs, global_step=..., is_train=True, **render_kwargs)`` followed by
run_sr.py's composite loss (run_sr.py:521-546, without nearclip), for DirectVoxGO and DirectMPIGO::

    loss, out = render_loss(model, rays_o, rays_d, viewdirs, target, global_step, render_kwargs)
    loss.backward()

The materialised path (train_forward.forward_samples) builds the flat sample list, compacts it with host syncs and
runs autograd through a few dozen ops; here the forward is one kernel plus a one-CTA loss reduction, and the backward
one kernel that re-marches every ray.  Nothing synchronises the host once the model's host-side constants are cached
(the first call on a model reads them).  The parameters are read live every call, never through the device scene of
the inference path.  The materialised path stays the one for custom losses, DirectContractedVoxGO and nearclip.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._scene import cached_host, host_float, linear_layers

LOSS_WEIGHTS = dict(main=1.0, entropy_last=0.01, distortion=0.01, rgbper=0.1)
TERMS = ('loss_main', 'loss_entropy_last', 'loss_distortion', 'loss_rgbper')
MAX_K0, MAX_WIDTH, MAX_DIM0, MAX_PE = 32, 128, 128, 10
_ACTS = {'relu': _lib.K4_ACT_RELU, 'gauss': _lib.K4_ACT_GAUSS, 'lkrelu': _lib.K4_ACT_LKRELU}


def _check_rays(name, t, n=None):
    if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f'render_loss: {name} must be an fp32 CUDA tensor [N,3]')
    if n is not None and t.shape[0] != n:
        raise ValueError(f'render_loss: {name} has {t.shape[0]} rows, rays_o has {n}')


def _weights(loss_weights):
    """The loss weights as given: a term left out of the dict has weight 0."""
    lw = {k: 0.0 for k in LOSS_WEIGHTS}
    for k, v in (loss_weights or {}).items():
        if k == 'nearclip':
            if v:
                raise NotImplementedError('render_loss: nearclip is DirectContractedVoxGO only; use the materialised path')
            continue
        if k not in lw:
            raise ValueError(f'render_loss: unknown loss weight {k!r}')
        lw[k] = float(v)
    if any(v < 0 for v in lw.values()):
        raise ValueError('render_loss: loss weights must be >= 0')
    return lw


def _model_shape(m):
    """(kind, act, layers) after the checks that reject what the kernels do not build."""
    kind = getattr(m, '_k4_kind', None)
    if kind == _lib.K4_KIND_DCVGO:
        raise NotImplementedError('render_loss: DirectContractedVoxGO trains on the materialised path')
    if kind not in (_lib.K4_KIND_DVGO, _lib.K4_KIND_DMPIGO):
        raise NotImplementedError(f'render_loss: {type(m).__name__} is not DirectVoxGO / DirectMPIGO')
    layers = linear_layers(m.rgbnet)
    act = getattr(m, 'act_type', 'relu') if kind == _lib.K4_KIND_DMPIGO else 'relu'
    if kind == _lib.K4_KIND_DMPIGO and layers and act not in _ACTS:
        raise NotImplementedError(f'render_loss: act_type {act!r}')
    C_ = int(m.k0.grid.shape[1])
    if layers:
        if len(layers) != 3:
            raise NotImplementedError('render_loss: the rgbnet must have 3 layers')
        if layers[0].out_features > MAX_WIDTH:
            raise NotImplementedError(f'render_loss: rgbnet width {layers[0].out_features} > {MAX_WIDTH}')
        if C_ > MAX_K0:
            raise NotImplementedError(f'render_loss: k0 has {C_} channels > {MAX_K0}')
        if layers[0].in_features > MAX_DIM0 or m.viewbase_pe > MAX_PE or getattr(m, 'spatial_pe', 0) > MAX_PE:
            raise NotImplementedError('render_loss: the rgbnet input is wider than the fp32 marcher mode accepts')
    elif C_ != 3:
        raise NotImplementedError('render_loss: a model without an rgbnet must have 3 k0 channels')
    return kind, act, layers


def _fill_args(m, kind, act, layers, kw, lw):
    a = _lib.TrainMarchArgs()
    a.kind = kind
    a.rgbnet_act = _ACTS[act] if layers else _lib.K4_ACT_RELU
    dens, k0 = m.density.grid, m.k0.grid
    a.world_size[:] = list(dens.shape[2:])
    a.k0_dim = int(k0.shape[1])
    mc = m.mask_cache
    a.mask_size[:] = list(mc.mask.shape)
    host = cached_host(m, 'train_fused', [m.xyz_min, m.xyz_max, mc.xyz2ijk_scale, mc.xyz2ijk_shift],
                       lambda: [t.detach().cpu().float().tolist() for t in (m.xyz_min, m.xyz_max, mc.xyz2ijk_scale,
                                                                            mc.xyz2ijk_shift)])
    a.xyz_min[:], a.xyz_max[:], a.xyz2ijk_scale[:], a.xyz2ijk_shift[:] = host
    a.fast_color_thres = float(m.fast_color_thres)
    a.near_ = float(kw['near'])
    a.stepsize = float(kw['stepsize'])
    a.bg = float(kw['bg'])
    a.max_world_size = int(max(dens.shape[2:]))
    vsr = m.voxel_size_ratio
    if torch.is_tensor(vsr):               # interval = float(stepsize * voxel_size_ratio), an fp32 product
        a.interval = float(np.float32(kw['stepsize']) * np.float32(host_float(m, 'voxel_size_ratio')))
    else:
        a.interval = float(kw['stepsize'] * vsr)
    if kind == _lib.K4_KIND_DVGO:
        a.act_shift = cached_host(m, 'act_shift', [m.act_shift], lambda: float(m.act_shift))
        a.voxel_size = host_float(m, 'voxel_size')
    else:
        if not (kw['near'] == 0 and kw['far'] == 1):             # lib/dmpigo.py:275
            raise ValueError('render_loss: DirectMPIGO renders with near = 0, far = 1')
        a.mpi_depth = int(m.mpi_depth)
    if layers:
        a.rgbnet_depth = 3
        a.rgbnet_width = int(layers[0].out_features)
        a.rgbnet_direct = int(bool(getattr(m, 'rgbnet_direct', True)))
        a.viewbase_pe = int(m.viewbase_pe)
        a.spatial_pe = int(getattr(m, 'spatial_pe', 0))
        if act == 'gauss':
            g = m.rgbnet[1]
            a.rgbnet_act_param = cached_host(m, 'gauss_a', [g.a], lambda: float(g.a))
    a.w_main, a.w_entropy = lw['main'], lw['entropy_last']
    a.w_distortion, a.w_rgbper = lw['distortion'], lw['rgbper']
    return a


class _RenderLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, keep, n, dev, *params):
        rgbm = torch.empty((n, 3), device=dev, dtype=torch.float32)
        T = torch.empty((n,), device=dev, dtype=torch.float32)
        loss = torch.empty((), device=dev, dtype=torch.float32)
        terms = torch.empty((4,), device=dev, dtype=torch.float32)
        ws = torch.empty(int(_lib.lib.k4_train_march_workspace_bytes(n)), device=dev, dtype=torch.uint8)
        a.d_rgb_marched, a.d_alphainv_last = rgbm.data_ptr(), T.data_ptr()
        a.d_loss, a.d_loss_terms = loss.data_ptr(), terms.data_ptr()
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(_lib.lib.k4_train_march_forward(C.byref(a), ws.data_ptr(), ws.numel(), C.c_void_p(stream)),
                   'k4_train_march_forward')
        ctx.a, ctx.keep, ctx.ws, ctx.dev = a, keep, ws, dev
        ctx.save_for_backward(*params)
        ctx.mark_non_differentiable(rgbm, T, terms)
        return loss, rgbm, T, terms

    @staticmethod
    def backward(ctx, g_loss, *_):
        params = ctx.saved_tensors
        need = ctx.needs_input_grad[4:]
        grads = [torch.zeros_like(p) if nd else None for p, nd in zip(params, need)]
        a = ctx.a
        ptr = lambda g: g.data_ptr() if g is not None else None
        a.d_grad_density, a.d_grad_k0 = ptr(grads[0]), ptr(grads[1])
        for i in range(3):
            a.d_grad_weight[i] = ptr(grads[2 + 2 * i]) if len(grads) > 2 else None
            a.d_grad_bias[i] = ptr(grads[3 + 2 * i]) if len(grads) > 2 else None
        g = g_loss.detach().to(torch.float32).contiguous()
        stream = torch.cuda.current_stream(ctx.dev).cuda_stream
        _lib.check(_lib.lib.k4_train_march_backward(C.byref(a), g.data_ptr(), ctx.ws.data_ptr(), ctx.ws.numel(),
                                                    C.c_void_p(stream)), 'k4_train_march_backward')
        return (None, None, None, None, *grads)


def render_loss(model, rays_o, rays_d, viewdirs, target, global_step, render_kwargs, loss_weights=LOSS_WEIGHTS):
    """The training forward and run_sr.py's composite loss (nearclip left out), fused.  Returns ``(loss, out)``:
    ``loss`` a 0-dim CUDA tensor whose backward accumulates into ``.grad`` of density.grid, k0.grid and the rgbnet's
    Linear weights and biases (whichever require grad); ``out`` holds detached ``rgb_marched [N,3]``,
    ``alphainv_last [N]`` and each weighted term (``loss_main``, ``loss_entropy_last``, ``loss_distortion``,
    ``loss_rgbper``) as a 0-dim tensor.  ``loss_weights`` is taken as given: a term it leaves out, or weights 0, is
    skipped (the default is run_sr.py's LLFF weights).  DirectMPIGO with
    ``render_kwargs['rand_bkgd']`` and a ``global_step`` draws its background with ``torch.rand((N, 3))``, as the
    training forward does."""
    kind, act, layers = _model_shape(model)
    lw = _weights(loss_weights)
    if kind == _lib.K4_KIND_DVGO and lw['distortion'] > 0:
        raise ValueError('render_loss: the distortion loss needs s / n_max, which DirectVoxGO does not return')
    _check_rays('rays_o', rays_o)
    n = rays_o.shape[0]
    if n < 1:
        raise ValueError('render_loss: no rays')
    for name, t in (('rays_d', rays_d), ('viewdirs', viewdirs), ('target', target)):
        _check_rays(name, t, n)
    dev = rays_o.device
    for t in (model.density.grid, model.k0.grid, model.mask_cache.mask):
        if t.device != dev:
            raise ValueError('render_loss: the model and the rays must be on the same device')
    a = _fill_args(model, kind, act, layers, render_kwargs, lw)
    a.n_rays = n
    keep = [t.contiguous() for t in (rays_o, rays_d, viewdirs, target)]
    a.d_rays_o, a.d_rays_d, a.d_viewdirs, a.d_target = (t.data_ptr() for t in keep)
    if kind == _lib.K4_KIND_DMPIGO and render_kwargs.get('rand_bkgd', False) and global_step is not None:
        bk = torch.rand((n, 3), device=dev)
        keep.append(bk)
        a.d_bkgd = bk.data_ptr()
    mask = model.mask_cache.mask
    mask = (mask.view(torch.uint8) if mask.dtype == torch.bool else mask.to(torch.uint8)).contiguous()
    keep.append(mask)
    a.d_mask = mask.data_ptr()
    params = [model.density.grid, model.k0.grid]
    for l in layers:
        params += [l.weight, l.bias]
    for p in params:
        if p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError('render_loss: the model parameters must be contiguous fp32')
    a.d_density, a.d_k0 = params[0].data_ptr(), params[1].data_ptr()
    for i, l in enumerate(layers):
        a.d_rgbnet_weight[i], a.d_rgbnet_bias[i] = l.weight.data_ptr(), l.bias.data_ptr()
    if kind == _lib.K4_KIND_DMPIGO:
        sg = model.act_shift.grid.detach().reshape(-1).contiguous()
        keep.append(sg)
        a.d_act_shift_grid = sg.data_ptr()
    with torch.cuda.device(dev):
        loss, rgbm, T, terms = _RenderLoss.apply(a, keep, n, dev, *params)
    out = {'rgb_marched': rgbm, 'alphainv_last': T}
    for i, k in enumerate(TERMS):
        out[k] = terms[i]
    return loss, out
