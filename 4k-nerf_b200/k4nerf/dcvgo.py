"""DirectContractedVoxGO (unbounded inward-facing scenes) with the reference constructor / checkpoint /
forward contract (lib/dcvgo.py:27-382), rendered by the fused marcher (contracted-space front-end of
csrc/k4_march.cu: per-step ray parameters, inf-norm contraction, cumdist_thres skipping, then the
same occupancy / density / alpha / colour / compositing chain).  SURVEY.md section 8(f-3)."""
import numpy as np
import torch
import torch.nn as nn

from . import _lib, grid, torch_efficient_distloss
from ._scene import FusedRenderMixin, cached_host, host_float
from .maintain import GridMaintenanceMixin
from .coarse import CoarseStageMixin


class DirectContractedVoxGO(FusedRenderMixin, GridMaintenanceMixin, CoarseStageMixin, nn.Module):
    _k4_kind = _lib.K4_KIND_DCVGO

    def __init__(self, xyz_min, xyz_max,
                 num_voxels=0, num_voxels_base=0,
                 alpha_init=None,
                 mask_cache_world_size=None,
                 fast_color_thres=0, bg_len=0.2,
                 contracted_norm='inf',
                 density_type='DenseGrid', k0_type='DenseGrid',
                 density_config={}, k0_config={},
                 rgbnet_dim=0,
                 rgbnet_depth=3, rgbnet_width=128,
                 viewbase_pe=4,
                 **kwargs):
        super().__init__()
        if contracted_norm != 'inf':
            raise NotImplementedError("only contracted_norm='inf' (the default) is built")
        xyz_min = torch.Tensor(xyz_min)
        xyz_max = torch.Tensor(xyz_max)
        assert len(((xyz_max - xyz_min) * 100000).long().unique()), 'scene bbox must be a cube in DirectContractedVoxGO'
        self.register_buffer('scene_center', (xyz_min + xyz_max) * 0.5)
        self.register_buffer('scene_radius', (xyz_max - xyz_min) * 0.5)
        self.register_buffer('xyz_min', torch.Tensor([-1, -1, -1]) - bg_len)
        self.register_buffer('xyz_max', torch.Tensor([1, 1, 1]) + bg_len)
        if isinstance(fast_color_thres, dict):
            self._fast_color_thres = fast_color_thres
            self.fast_color_thres = fast_color_thres[0]
        else:
            self._fast_color_thres = None
            self.fast_color_thres = fast_color_thres
        self.bg_len = bg_len
        self.contracted_norm = contracted_norm
        self.num_voxels_base = num_voxels_base
        self.voxel_size_base = ((self.xyz_max - self.xyz_min).prod() / self.num_voxels_base).pow(1 / 3)
        self._set_grid_resolution(num_voxels)
        self.alpha_init = alpha_init
        self.register_buffer('act_shift', torch.FloatTensor([np.log(1 / (1 - alpha_init) - 1)]))
        self.density_type, self.density_config = density_type, density_config
        self.k0_type, self.k0_config = k0_type, k0_config
        self.density = grid.create_grid(density_type, channels=1, world_size=self.world_size,
                                        xyz_min=self.xyz_min, xyz_max=self.xyz_max, config=density_config)
        self.rgbnet_kwargs = {'rgbnet_dim': rgbnet_dim, 'rgbnet_depth': rgbnet_depth, 'rgbnet_width': rgbnet_width,
                              'viewbase_pe': viewbase_pe}
        self.viewbase_pe = viewbase_pe
        if rgbnet_dim <= 0:
            self.k0_dim = 3
            self.rgbnet = None
        else:
            self.k0_dim = rgbnet_dim
            self.register_buffer('viewfreq', torch.FloatTensor([(2 ** i) for i in range(viewbase_pe)]))
            dim0 = (3 + 3 * viewbase_pe * 2) + self.k0_dim
            self.rgbnet = nn.Sequential(
                nn.Linear(dim0, rgbnet_width), nn.ReLU(inplace=True),
                *[nn.Sequential(nn.Linear(rgbnet_width, rgbnet_width), nn.ReLU(inplace=True)) for _ in range(rgbnet_depth - 2)],
                nn.Linear(rgbnet_width, 3),
            )
            nn.init.constant_(self.rgbnet[-1].bias, 0)
        self.k0 = grid.create_grid(k0_type, channels=self.k0_dim, world_size=self.world_size,
                                   xyz_min=self.xyz_min, xyz_max=self.xyz_max, config=k0_config)
        if mask_cache_world_size is None:
            mask_cache_world_size = self.world_size
        mask = torch.ones([int(w) for w in mask_cache_world_size], dtype=torch.bool)
        self.mask_cache = grid.MaskGrid(path=None, mask=mask, xyz_min=self.xyz_min, xyz_max=self.xyz_max)

    def _set_grid_resolution(self, num_voxels):
        # lib/dcvgo.py:130-141
        self.num_voxels = num_voxels
        self.voxel_size = ((self.xyz_max - self.xyz_min).prod() / num_voxels).pow(1 / 3)
        self.world_size = ((self.xyz_max - self.xyz_min) / self.voxel_size).long()
        self.world_len = self.world_size[0].item()
        self.voxel_size_ratio = self.voxel_size / self.voxel_size_base

    def get_kwargs(self):
        return {
            'xyz_min': self.xyz_min.cpu().numpy(), 'xyz_max': self.xyz_max.cpu().numpy(),
            'num_voxels': self.num_voxels, 'num_voxels_base': self.num_voxels_base,
            'alpha_init': self.alpha_init, 'voxel_size_ratio': self.voxel_size_ratio,
            'mask_cache_world_size': list(self.mask_cache.mask.shape),
            'fast_color_thres': self.fast_color_thres, 'contracted_norm': self.contracted_norm,
            'density_type': self.density_type, 'k0_type': self.k0_type,
            'density_config': self.density_config, 'k0_config': self.k0_config,
            **self.rgbnet_kwargs,
        }

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        for name, mod in (('density', self.density), ('k0', self.k0)):
            key = prefix + name + '.grid'
            if key in state_dict and state_dict[key].shape != mod.grid.shape:
                mod.grid = nn.Parameter(torch.zeros_like(state_dict[key]))
        key = prefix + 'mask_cache.mask'
        if key in state_dict and state_dict[key].shape != self.mask_cache.mask.shape:
            self.mask_cache.mask = torch.zeros_like(state_dict[key])
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
        self.world_size = torch.tensor(list(self.density.grid.shape[2:]), dtype=torch.long)
        self.world_len = int(self.world_size[0])
        self.invalidate_scene()

    def forward(self, rays_o, rays_d, viewdirs, global_step=None, is_train=False, **render_kwargs):
        """lib/dcvgo.py:262-382.  The dict-valued fast_color_thres schedule (lib/dcvgo.py:269-271) is applied
        here; the threshold is baked into the device scene, whose fingerprint sees the change."""
        if isinstance(self._fast_color_thres, dict) and global_step in self._fast_color_thres:
            print(f'dcvgo: update fast_color_thres {self.fast_color_thres} => {self._fast_color_thres[global_step]}')
            self.fast_color_thres = self._fast_color_thres[global_step]
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            from .train_forward import forward_samples
            return forward_samples(self, rays_o, rays_d, viewdirs, global_step=global_step, is_train=is_train, **render_kwargs)
        return super().forward(rays_o, rays_d, viewdirs, global_step=global_step, **render_kwargs)

    def resolve_mlp_mode(self, mode):
        if mode == 'tc':
            return 'ws'        # the contracted front-end is built into the warp-specialised kernel only
        return super().resolve_mlp_mode(mode)

    def _scene_extra(self):
        bufs = [self.act_shift, self.scene_center, self.scene_radius]
        act, center, radius = cached_host(self, 'scene_host', bufs, lambda: (
            float(self.act_shift), self.scene_center.detach().cpu().tolist(), self.scene_radius.detach().cpu().tolist()))
        return {
            'act_shift': act, 'voxel_size': host_float(self, 'voxel_size'), 'rgbnet_direct': True,
            'viewbase_pe': self.viewbase_pe if self.rgbnet is not None else 0,
            'scene_center': center, 'scene_radius': radius,
            'bg_len': float(self.bg_len), 'world_len': int(self.world_len),
        }

    def sample_t(self, stepsize, device):
        """The per-step ray parameters of sample_ray (lib/dcvgo.py:239-248), same torch expressions."""
        N_inner = int(2 / (2 + 2 * self.bg_len) * self.world_len / stepsize) + 1
        N_outer = N_inner
        b_inner = torch.linspace(0, 2, N_inner + 1, device=device)
        b_outer = 2 / torch.linspace(1, 1 / 128, N_outer + 1, device=device)
        return torch.cat([(b_inner[1:] + b_inner[:-1]) * 0.5, (b_outer[1:] + b_outer[:-1]) * 0.5]).contiguous()

    def _extra_render_args(self, a, render_kwargs, device, keep):
        t = self.sample_t(render_kwargs['stepsize'], device)
        keep.append(t)
        a.d_t_list = t.data_ptr()
        a.n_t = int(t.numel())
        a.dist_thres = float((2 + 2 * self.bg_len) / self.world_len * render_kwargs['stepsize'] * 0.95)   # lib/dcvgo.py:283


class DistortionLoss(torch.autograd.Function):
    """lib/dcvgo.py:385-407 with the reference's signature (w, s, n_max, ray_id), on the kernels of
    ``torch_efficient_distloss.flatten_eff_distloss``.  The forward is that loss with interval = 1 / n_max.

    The backward reproduces lib/dcvgo.py:406 as written: ``grad_back * (grad_bi + grad_uni)`` with no division by
    n = ray_id.max() + 1, so the gradient it returns is n times the gradient of its own forward (the reference's
    quirk, kept so that a training loop that uses it behaves as it does with the reference).  Only w receives one."""

    @staticmethod
    def forward(ctx, w, s, n_max, ray_id):
        return torch_efficient_distloss.autograd_forward(ctx, w, s, 1 / n_max, ray_id, divide_by_n=False)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_back):
        return torch_efficient_distloss.autograd_backward(ctx, grad_back)


distortion_loss = DistortionLoss.apply
