"""DirectMPIGO with the reference constructor / checkpoint / forward contract (lib/dmpigo.py:18-427),
rendered by the fused sm_90a marcher."""
import numpy as np
import torch
import torch.nn as nn

from . import _lib, grid
from .act import GaussianActivation

# act_type -> the module after every hidden nn.Linear of the rgbnet (lib/dmpigo.py:89-95) and its K4_ACT_* code
_ACT_TYPES = {'relu': _lib.K4_ACT_RELU, 'gauss': _lib.K4_ACT_GAUSS, 'lkrelu': _lib.K4_ACT_LKRELU}


def make_act(act_type):
    if act_type == 'relu':
        return nn.ReLU(inplace=True)
    if act_type == 'gauss':
        return GaussianActivation(a=0.05)
    if act_type == 'lkrelu':
        return nn.LeakyReLU()
    raise ValueError(f"act_type must be one of 'relu', 'gauss', 'lkrelu', not {act_type!r}")
from ._scene import FusedRenderMixin
from .maintain import GridMaintenanceMixin
from .coarse import CoarseStageMixin


class DirectMPIGO(FusedRenderMixin, GridMaintenanceMixin, CoarseStageMixin, nn.Module):
    _k4_kind = _lib.K4_KIND_DMPIGO

    def __init__(self, xyz_min, xyz_max,
                 num_voxels=0, mpi_depth=0,
                 mask_cache_path=None, mask_cache_thres=1e-3, mask_cache_world_size=None,
                 fast_color_thres=0,
                 density_type='DenseGrid', k0_type='DenseGrid',
                 density_config={}, k0_config={},
                 rgbnet_dim=0,
                 rgbnet_depth=3, rgbnet_width=128,
                 viewbase_pe=0, spatial_pe=0,
                 **kwargs):
        super().__init__()
        self.register_buffer('xyz_min', torch.Tensor(xyz_min))
        self.register_buffer('xyz_max', torch.Tensor(xyz_max))
        self.fast_color_thres = fast_color_thres
        self._set_grid_resolution(num_voxels, mpi_depth)
        self.density_type, self.density_config = density_type, density_config
        self.k0_type, self.k0_config = k0_type, k0_config
        self.density = grid.create_grid(density_type, channels=1, world_size=self.world_size,
                                        xyz_min=self.xyz_min, xyz_max=self.xyz_max, config=density_config)
        # depth-dependent density bias, lib/dmpigo.py:48-58
        self.act_shift = grid.DenseGrid(channels=1, world_size=[1, 1, mpi_depth], xyz_min=xyz_min, xyz_max=xyz_max)
        self.act_shift.grid.requires_grad = False
        with torch.no_grad():
            g = np.full([mpi_depth], 1. / mpi_depth - 1e-6)
            p = [1 - g[0]]
            for i in range(1, len(g)):
                p.append((1 - g[:i + 1].sum()) / (1 - g[:i].sum()))
            for i in range(len(p)):
                self.act_shift.grid[..., i].fill_(np.log(p[i] ** (-1 / self.voxel_size_ratio) - 1))

        self.rgbnet_kwargs = {
            'rgbnet_dim': rgbnet_dim, 'rgbnet_depth': rgbnet_depth, 'rgbnet_width': rgbnet_width,
            'viewbase_pe': viewbase_pe, 'spatial_pe': spatial_pe,
        }
        self.viewbase_pe, self.spatial_pe = viewbase_pe, spatial_pe
        self.dim_rend = 3
        self.act_type = kwargs.get('act_type', 'relu')
        self.mode_type = kwargs.get('mode_type', 'mlp')
        if rgbnet_dim <= 0:
            self.k0_dim = 3
            self.rgbnet = None
        else:
            if self.mode_type in ('TRANS', 'adain'):
                raise NotImplementedError('mode_type TRANS/adain need modules the reference does not ship')
            self.k0_dim = rgbnet_dim
            self.register_buffer('viewfreq', torch.FloatTensor([(2 ** i) for i in range(viewbase_pe)]))
            self.register_buffer('posfreq', torch.FloatTensor([(2 ** i) for i in range(spatial_pe)]))
            self.dim0 = (3 + 3 * viewbase_pe * 2 + 3 + 3 * spatial_pe * 2) + self.k0_dim
            self.pe_dim = 3 + 3 * viewbase_pe * 2 + 3 + 3 * spatial_pe * 2
            act = make_act(self.act_type)      # ONE instance after every hidden Linear, as the reference shares it
            self.rgbnet = nn.Sequential(
                nn.Linear(self.dim0, rgbnet_width), act,
                *[nn.Sequential(nn.Linear(rgbnet_width, rgbnet_width), act) for _ in range(rgbnet_depth - 2)],
                nn.Linear(rgbnet_width, self.dim_rend),
            )
            nn.init.constant_(self.rgbnet[-1].bias, 0)
        self.k0 = grid.create_grid(k0_type, channels=self.k0_dim, world_size=self.world_size,
                                   xyz_min=self.xyz_min, xyz_max=self.xyz_max, config=k0_config)

        self.mask_cache_path = mask_cache_path
        self.mask_cache_thres = mask_cache_thres
        if mask_cache_world_size is None:
            mask_cache_world_size = self.world_size
        if mask_cache_path:
            from .maintain import mask_from_coarse_checkpoint
            mask = mask_from_coarse_checkpoint(mask_cache_path, mask_cache_thres, self.xyz_min, self.xyz_max, mask_cache_world_size)
        else:
            mask = torch.ones([int(w) for w in mask_cache_world_size], dtype=torch.bool)
        self.mask_cache = grid.MaskGrid(path=None, mask=mask, xyz_min=self.xyz_min, xyz_max=self.xyz_max)

    def _set_grid_resolution(self, num_voxels, mpi_depth):
        # lib/dmpigo.py:156-164
        self.num_voxels = num_voxels
        self.mpi_depth = mpi_depth
        r = (num_voxels / self.mpi_depth / (self.xyz_max - self.xyz_min)[:2].prod()).sqrt()
        self.world_size = torch.zeros(3, dtype=torch.long)
        self.world_size[:2] = (self.xyz_max - self.xyz_min)[:2] * r
        self.world_size[2] = self.mpi_depth
        self.voxel_size_ratio = 256. / mpi_depth

    # ---- grid maintenance (maintain.py) specifics of the MPI model ----
    _k4_shift_in_alpha = False          # activate_density: Raw2Alpha(density, 0, interval), lib/dmpigo.py:258-261

    def _rescaled_density_for_mask(self):
        return self.density.get_dense_grid() + self.act_shift.grid           # lib/dmpigo.py:205

    def _tv_weights(self, weight):
        wxy = weight * self.world_size[:2].max() / 128                       # lib/dmpigo.py:247-255
        wz = weight * self.mpi_depth / 128
        return wxy, wxy, wz

    def get_kwargs(self):
        return {
            'xyz_min': self.xyz_min.cpu().numpy(), 'xyz_max': self.xyz_max.cpu().numpy(),
            'num_voxels': self.num_voxels, 'mpi_depth': self.mpi_depth,
            'voxel_size_ratio': self.voxel_size_ratio,
            'mask_cache_path': self.mask_cache_path, 'mask_cache_thres': self.mask_cache_thres,
            'mask_cache_world_size': list(self.mask_cache.mask.shape),
            'fast_color_thres': self.fast_color_thres,
            'density_type': self.density_type, 'k0_type': self.k0_type,
            'density_config': self.density_config, 'k0_config': self.k0_config,
            'mode_type': self.mode_type, 'act_type': self.act_type, 'dim_rend': self.dim_rend,
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
        self.invalidate_scene()

    def _scene_extra(self):
        return {
            'mpi_depth': int(self.mpi_depth), 'act_shift_grid': self.act_shift.grid.detach(),
            'viewbase_pe': self.viewbase_pe if self.rgbnet is not None else 0,
            'spatial_pe': self.spatial_pe if self.rgbnet is not None else 0,
            'rgbnet_act': _ACT_TYPES[self.act_type] if self.rgbnet is not None else _lib.K4_ACT_RELU,
            'rgbnet_act_param': self.rgbnet[1].a.detach() if self.rgbnet is not None and self.act_type == 'gauss' else None,
        }
