"""Device-scene handle management shared by DirectVoxGO / DirectMPIGO.

A ``k4_scene`` (include/k4nerf.h) is an immutable, repacked device copy of a model's tensors.  The
modules rebuild it lazily whenever a parameter/buffer was modified in place or moved
(tensor ``_version`` / ``data_ptr`` fingerprint), so ``load_state_dict`` and ``.to(device)`` just work.
"""
import ctypes as C

import torch

from . import _lib

_DEFAULT_MLP_MODE = 'auto'     # warp-specialised wgmma kernel when the shape has a build, else mma.sync f16, else fp32


class SceneHandle:
    def __init__(self, ptr, device, fingerprint):
        self.ptr = ptr
        self.device = device
        self.fingerprint = fingerprint

    def __del__(self):
        try:
            if self.ptr:
                _lib.lib.k4_scene_destroy(self.ptr)
                self.ptr = None
        except Exception:
            pass


def _fp(tensors):
    return tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in tensors if t is not None)


def cached_host(module, name, tensors, fn):
    """Host copies of small device buffers (act_shift, scene centre ...) cached by the buffers'
    (data_ptr, _version): float(buffer) is a device->host copy + stream sync, which must not happen on
    every render call."""
    cache = module.__dict__.setdefault('_k4_hostcache', {})
    fp = _fp(tensors)
    e = cache.get(name)
    if e is None or e[0] != fp:
        e = (fp, fn())
        cache[name] = e
    return e[1]


def host_float(module, name):
    """float(module.<name>) without a per-call device sync when the attribute is a CUDA tensor (voxel_size /
    voxel_size_ratio become CUDA tensors once _set_grid_resolution runs after .to(device))."""
    v = getattr(module, name)
    if torch.is_tensor(v) and v.is_cuda:
        return cached_host(module, 'f:' + name, [v], lambda: float(v))
    return float(v)


def scalar_fingerprint(module, extra):
    """Scalars baked into the device scene (k4_scene_desc): a change must rebuild it."""
    return (float(module.fast_color_thres), host_float(module, 'voxel_size_ratio'), float(extra.get('act_shift', 0.0)),
            float(extra.get('voxel_size', 0.0)), int(extra.get('viewbase_pe', 0)), int(extra.get('spatial_pe', 0)),
            bool(extra.get('rgbnet_direct', True)), int(extra.get('rgbnet_act', _lib.K4_ACT_RELU)))


def require_cuda(*tensors):
    for t in tensors:
        if not t.is_cuda:
            # mirrors CHECK_CUDA of the reference extension (lib/cuda/render_utils.cpp:46)
            raise RuntimeError('k4nerf: tensors must be CUDA tensors (there is no CPU path)')


def linear_layers(rgbnet):
    """The nn.Linear modules of the reference's rgbnet Sequential, in order (lib/dvgo.py:116-123)."""
    if rgbnet is None:
        return []
    return [m for m in rgbnet.modules() if isinstance(m, torch.nn.Linear)]


def gather_tensors(module, extra):
    """Every tensor the device scene is derived from (live objects, for change detection)."""
    mc = module.mask_cache
    layers = linear_layers(module.rgbnet)
    tensors = [module.density.grid, module.k0.grid, mc.mask, mc.xyz2ijk_scale, mc.xyz2ijk_shift,
               module.xyz_min, module.xyz_max]
    tensors += [p for l in layers for p in (l.weight, l.bias)]
    if extra.get('act_shift_grid') is not None:
        tensors.append(extra['act_shift_grid'])
    if extra.get('rgbnet_act_param') is not None:
        tensors.append(extra['rgbnet_act_param'])
    return tensors


def build_scene(kind, module, extra):
    """Create the device scene for ``module`` (DirectVoxGO / DirectMPIGO)."""
    density = module.density.grid.detach()
    k0 = module.k0.grid.detach()
    mc = module.mask_cache
    layers = linear_layers(module.rgbnet)
    require_cuda(density, k0, mc.mask)
    fingerprint = (_fp(gather_tensors(module, extra)), scalar_fingerprint(module, extra))
    dev = density.device
    d = _lib.SceneDesc()
    d.kind = kind
    X, Y, Z = density.shape[2:]
    d.world_size[:] = [X, Y, Z]
    d.k0_dim = k0.shape[1]
    d.mask_size[:] = list(mc.mask.shape)
    d.xyz_min[:] = module.xyz_min.detach().cpu().tolist()
    d.xyz_max[:] = module.xyz_max.detach().cpu().tolist()
    d.xyz2ijk_scale[:] = mc.xyz2ijk_scale.detach().cpu().tolist()
    d.xyz2ijk_shift[:] = mc.xyz2ijk_shift.detach().cpu().tolist()
    d.act_shift = float(extra.get('act_shift', 0.0))
    d.voxel_size = float(extra.get('voxel_size', 0.0))
    d.voxel_size_ratio = host_float(module, 'voxel_size_ratio')
    d.fast_color_thres = float(module.fast_color_thres)
    d.max_world_size = int(max(X, Y, Z))
    d.mpi_depth = int(extra.get('mpi_depth', 0))
    d.rgbnet_depth = len(layers)
    d.rgbnet_width = int(layers[0].out_features) if layers else 0
    d.rgbnet_direct = int(bool(extra.get('rgbnet_direct', True)))
    d.viewbase_pe = int(extra.get('viewbase_pe', 0))
    d.spatial_pe = int(extra.get('spatial_pe', 0))
    d.rgbnet_act = int(extra.get('rgbnet_act', _lib.K4_ACT_RELU))
    if extra.get('rgbnet_act_param') is not None:
        d.rgbnet_act_param = float(extra['rgbnet_act_param'])      # GaussianActivation.a, read when the scene is built
    if 'scene_center' in extra:
        d.scene_center[:] = extra['scene_center']
        d.scene_radius[:] = extra['scene_radius']
        d.bg_len = float(extra['bg_len'])
        d.world_len = int(extra['world_len'])
    keep = []

    def dptr(t, dtype):
        t = t.detach().to(device=dev, dtype=dtype).contiguous()
        keep.append(t)
        return t.data_ptr()

    d.d_density = dptr(density, torch.float32)
    d.d_k0 = dptr(k0, torch.float32)
    d.d_mask = dptr(mc.mask, torch.uint8) if mc.mask.dtype != torch.bool else dptr(mc.mask.view(torch.uint8), torch.uint8)
    if extra.get('act_shift_grid') is not None:
        d.d_act_shift_grid = dptr(extra['act_shift_grid'].reshape(-1), torch.float32)
    for i, l in enumerate(layers):
        d.d_rgbnet_weight[i] = dptr(l.weight, torch.float32)
        d.d_rgbnet_bias[i] = dptr(l.bias, torch.float32)
    out = C.c_void_p()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        _lib.check(_lib.lib.k4_scene_create(C.byref(d), C.c_void_p(stream.cuda_stream), C.byref(out)),
                   'k4_scene_create')
        stream.synchronize()        # the repack kernels read `keep`; creation is a one-off
    return SceneHandle(out.value, dev, fingerprint)


class FusedRenderMixin:
    """forward() of both scene models: one k4_render_rays call."""
    mlp_mode = _DEFAULT_MLP_MODE

    def _scene_extra(self):
        raise NotImplementedError

    def _extra_render_args(self, a, render_kwargs, device, keep):
        """Hook for model-specific k4_render_args fields (DirectContractedVoxGO's step list)."""

    def _get_scene(self):
        h = getattr(self, '_k4_handle', None)
        extra = self._scene_extra()
        if h is not None and (_fp(gather_tensors(self, extra)), scalar_fingerprint(self, extra)) == h.fingerprint:
            return h
        h = build_scene(self._k4_kind, self, extra)
        object.__setattr__(self, '_k4_handle', h)
        return h

    def resolve_mlp_mode(self, mode):
        """'auto' -> the fastest mode built for this model's shape (every mode is checked against the fp32
        oracle by tests/test_gpu_marcher.py).  'tc' / 'tcgen05' name the wgmma marcher, 'ws'."""
        if mode in ('tc', 'tcgen05'):
            return 'ws'
        if mode != 'auto':
            return mode
        if not linear_layers(self.rgbnet):
            return 'fp32'
        best = _lib.lib.k4_scene_best_mlp_mode(self._get_scene().ptr)       # the library knows which shapes have a wgmma build
        return {_lib.K4_MLP_TCGEN05_WS: 'ws', _lib.K4_MLP_F16: 'f16'}.get(best, 'fp32')

    def invalidate_scene(self):
        object.__setattr__(self, '_k4_handle', None)

    @torch.no_grad()
    def render_rays(self, rays_o, rays_d, viewdirs, render_kwargs, image_hw=None, mlp_mode=None,
                    debug=False, out=None, phases=None):
        """Run the fused kernel.  Returns dict(rgb_marched, alphainv_last[, depth][, ray_stats, t_minmax, counters]).
        ``out``: optional dict of caller-owned contiguous fp32 CUDA tensors ``rgb_marched [N,3]``, ``alphainv_last [N]``
        (and ``depth [N]``) the kernel writes into -- e.g. views of a packed communication buffer (k4nerf.dist) -- or a
        :class:`k4nerf.dist.FrameTarget`: the rays are one rank's rows of a block-cyclic multi-GPU frame and every ray is
        stored straight into every rank's image-order frame (k4_render_rays_frames); the returned dict then holds only
        the debug outputs.
        ``phases``: a contiguous int64 CUDA tensor [max_ctas, 4, K4_PHASE_SLOTS]; the 'ws' kernel then runs in its profiled
        instantiation (k4_testing_march_phases), which fills the tensor's first ``ret['n_ctas']`` rows with the phase
        cycles of every warpgroup."""
        assert rays_o.dim() == 2 and rays_o.shape[-1] == 3, 'Only suuport point queries in [N, 3] format'
        require_cuda(rays_o, rays_d, viewdirs)
        h = self._get_scene()
        dev = h.device
        rays_o = rays_o.to(torch.float32).contiguous()
        rays_d = rays_d.to(torch.float32).contiguous()
        viewdirs = viewdirs.to(torch.float32).contiguous()
        N = rays_o.shape[0]
        want_depth = bool(render_kwargs.get('render_depth', False))
        frames = getattr(out, 'frame_dst', None)
        if frames is not None:
            if N % int(frames.frame_w) != 0:
                raise ValueError('render_rays(out=FrameTarget): the rays must be whole rows of the frame')
            rgb = alphainv = depth = None
        elif out is not None:
            rgb, alphainv, depth = out['rgb_marched'], out['alphainv_last'], (out.get('depth') if want_depth else None)
            for t, shp in ((rgb, (N, 3)), (alphainv, (N,)), (depth, (N,))):
                if t is not None and not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shp):
                    raise ValueError('render_rays(out=...): outputs must be contiguous fp32 CUDA tensors of shape [N,3] / [N]')
            want_depth = depth is not None
        else:
            rgb = torch.empty((N, 3), device=dev, dtype=torch.float32)
            alphainv = torch.empty((N,), device=dev, dtype=torch.float32)
            depth = torch.empty((N,), device=dev, dtype=torch.float32) if want_depth else None
        a = _lib.RenderArgs()
        a.near_ = float(render_kwargs['near'])
        a.far_ = float(render_kwargs['far'])
        a.stepsize = float(render_kwargs['stepsize'])
        a.bg = float(render_kwargs['bg'])
        a.render_depth = int(want_depth)
        a.mlp_mode = _lib.MLP_MODES[self.resolve_mlp_mode(mlp_mode or self.mlp_mode)]
        if image_hw is not None and image_hw[0] * image_hw[1] == N:
            a.image_h, a.image_w = int(image_hw[0]), int(image_hw[1])
        keep = []
        self._extra_render_args(a, render_kwargs, dev, keep)
        o = _lib.RenderOut()
        if frames is None:
            o.d_rgb_marched = rgb.data_ptr()
            o.d_alphainv_last = alphainv.data_ptr()
            o.d_depth = depth.data_ptr() if depth is not None else None
            ret = {'rgb_marched': rgb, 'alphainv_last': alphainv}
            if depth is not None:
                ret['depth'] = depth
        else:
            ret = {}
        if debug:
            ret['ray_stats'] = torch.zeros((N, 4), device=dev, dtype=torch.int32)
            ret['t_minmax'] = torch.zeros((N, 2), device=dev, dtype=torch.float32)
            ret['counters'] = torch.zeros((4,), device=dev, dtype=torch.int64)
            o.d_ray_stats = ret['ray_stats'].data_ptr()
            o.d_t_minmax = ret['t_minmax'].data_ptr()
            o.d_counters = ret['counters'].data_ptr()
        if N == 0:
            return ret
        ws_bytes = _lib.lib.k4_render_workspace_bytes(h.ptr, N)
        ws = getattr(self, '_k4_ws', None)
        if ws is None or ws.numel() < ws_bytes or ws.device != dev:
            ws = torch.empty(int(ws_bytes), device=dev, dtype=torch.uint8)
            object.__setattr__(self, '_k4_ws', ws)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            if phases is not None:
                if frames is not None or not (phases.is_cuda and phases.dtype == torch.int64 and phases.is_contiguous()
                                              and phases.dim() == 3 and tuple(phases.shape[1:]) == (4, _lib.K4_PHASE_SLOTS)):
                    raise ValueError('render_rays(phases=...): an int64 CUDA tensor [max_ctas, 4, K4_PHASE_SLOTS], no FrameTarget')
                n_ctas = C.c_int32(0)
                _lib.check(_lib.lib.k4_testing_march_phases(h.ptr, C.byref(a), rays_o.data_ptr(), rays_d.data_ptr(),
                                                            viewdirs.data_ptr(), N, C.byref(o), ws.data_ptr(), ws.numel(),
                                                            phases.data_ptr(), phases.shape[0], C.byref(n_ctas),
                                                            C.c_void_p(stream)), 'k4_testing_march_phases')
                ret['n_ctas'] = n_ctas.value
            elif frames is not None:
                _lib.check(_lib.lib.k4_render_rays_frames(h.ptr, C.byref(a), rays_o.data_ptr(), rays_d.data_ptr(),
                                                          viewdirs.data_ptr(), N, C.byref(frames), C.byref(o), ws.data_ptr(),
                                                          ws.numel(), C.c_void_p(stream)), 'k4_render_rays_frames')
            else:
                _lib.check(_lib.lib.k4_render_rays(h.ptr, C.byref(a), rays_o.data_ptr(), rays_d.data_ptr(),
                                                   viewdirs.data_ptr(), N, C.byref(o), ws.data_ptr(),
                                                   ws.numel(), C.c_void_p(stream)), 'k4_render_rays')
        return ret

    def forward(self, rays_o, rays_d, viewdirs, global_step=None, **render_kwargs):
        """Volume rendering -- the reference's forward contract at inference
        (lib/dvgo.py:327-448, lib/dmpigo.py:292-427).

        Returns ``alphainv_last [N]``, ``rgb_marched [N,3]``, ``rgb_feature`` (the SAME tensor: the
        reference aliases it and adds the background in place, lib/dvgo.py:425-427) and ``depth [N]``
        when ``render_kwargs['render_depth']``.  The flat per-sample lists the reference also returns
        (``weights``, ``raw_alpha``, ``raw_rgb``, ``ray_id``, ``s``) are training-only and are never
        materialised by the fused kernel; with autograd enabled (training) the call is routed to
        ``train_forward.forward_samples``, which returns them.
        """
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training: the materialised, differentiable pipeline on the op-level kernels (section 8 f-2)
            from .train_forward import forward_samples
            return forward_samples(self, rays_o, rays_d, viewdirs, global_step=global_step, **render_kwargs)
        ret = self.render_rays(rays_o, rays_d, viewdirs, render_kwargs)
        ret['rgb_feature'] = ret['rgb_marched']
        return ret
