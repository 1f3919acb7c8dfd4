"""Restatement of the reference's scene-model forward passes -- TEST INFRASTRUCTURE ONLY.

``dvgo_forward``   follows DirectVoxGO.forward   (lib/dvgo.py:327-448, sample_ray :295-325)
``dmpigo_forward`` follows DirectMPIGO.forward   (lib/dmpigo.py:292-427, sample_ray :263-290)
``dense_grid``     follows DenseGrid.forward     (lib/grid.py:117-128)
``mask_grid``      follows MaskGrid.forward      (lib/grid.py:295-304)
``dvgo_state`` / ``dmpigo_state`` restate the constructors' arithmetic
                   (lib/dvgo.py:36-46,152-158; lib/dmpigo.py:36-58,156-164; lib/grid.py:291-293).

The pipeline keeps the reference's structure on purpose: flat ``[M]`` point lists, boolean-mask
compaction after every stage, ``F.grid_sample`` for interpolation, ``nn.Linear``-equivalent
``F.linear`` for the MLP and ``index_add_`` for ``torch_scatter.segment_coo(reduce='sum')``
(sorted index, lib/dvgo.py:415).  The custom ops come from an ``ops`` backend (oracle/ops.py):
``CpuOps`` (C restatement) or ``RefExtOps`` (the reference's own kernels, GPU box only).

A model is a plain ``dict`` of tensors/scalars ("state"), not an nn.Module, so that this file
shares no code with the product package.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------
# constructors' arithmetic
# ----------------------------------------------------------------------------------------------
def mask_grid_state(mask, xyz_min, xyz_max):
    """lib/grid.py:286-293: xyz2ijk_scale = (shape-1)/(max-min); shift = -min*scale."""
    xyz_min = torch.as_tensor(xyz_min, dtype=torch.float32)
    xyz_max = torch.as_tensor(xyz_max, dtype=torch.float32)
    xyz_len = xyz_max - xyz_min
    scale = (torch.Tensor(list(mask.shape)) - 1) / xyz_len
    shift = -xyz_min * scale
    return {'mask': mask.bool(), 'xyz2ijk_scale': scale, 'xyz2ijk_shift': shift}


def dvgo_state(xyz_min, xyz_max, num_voxels, num_voxels_base, alpha_init, fast_color_thres,
               rgbnet_dim=0, rgbnet_direct=False, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4,
               mask_cache_world_size=None):
    """Shapes and derived scalars of DirectVoxGO.__init__ (lib/dvgo.py:24-150), zero-filled grids."""
    st = {'kind': 'dvgo'}
    st['xyz_min'] = torch.Tensor(xyz_min)
    st['xyz_max'] = torch.Tensor(xyz_max)
    st['fast_color_thres'] = fast_color_thres
    # lib/dvgo.py:42,155-158
    st['voxel_size_base'] = ((st['xyz_max'] - st['xyz_min']).prod() / num_voxels_base).pow(1 / 3)
    st['act_shift'] = torch.FloatTensor([np.log(1 / (1 - alpha_init) - 1)])
    st['voxel_size'] = ((st['xyz_max'] - st['xyz_min']).prod() / num_voxels).pow(1 / 3)
    st['world_size'] = ((st['xyz_max'] - st['xyz_min']) / st['voxel_size']).long()
    st['max_world_size'] = st['world_size'].max()
    st['voxel_size_ratio'] = st['voxel_size'] / st['voxel_size_base']
    ws = st['world_size'].tolist()
    st['density'] = torch.zeros([1, 1, *ws])
    st['rgbnet_dim'] = rgbnet_dim
    st['rgbnet_direct'] = rgbnet_direct
    if rgbnet_dim <= 0:
        st['k0_dim'] = 3
        st['rgbnet'] = None
    else:
        st['k0_dim'] = rgbnet_dim
        st['viewfreq'] = torch.FloatTensor([(2 ** i) for i in range(viewbase_pe)])
        dim0 = 3 + 3 * viewbase_pe * 2
        dim0 += st['k0_dim'] if rgbnet_direct else st['k0_dim'] - 3
        st['dim0'] = dim0
        dims = [dim0] + [rgbnet_width] * (rgbnet_depth - 1) + [3]
        st['rgbnet'] = [(torch.zeros(dims[i + 1], dims[i]), torch.zeros(dims[i + 1])) for i in range(len(dims) - 1)]
    st['k0'] = torch.zeros([1, st['k0_dim'], *ws])
    if mask_cache_world_size is None:
        mask_cache_world_size = ws
    st['mask_cache'] = mask_grid_state(torch.ones(list(mask_cache_world_size), dtype=torch.bool),
                                       st['xyz_min'], st['xyz_max'])
    return st


def dmpigo_state(xyz_min, xyz_max, num_voxels, mpi_depth, fast_color_thres,
                 rgbnet_dim=0, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=0, spatial_pe=0,
                 mask_cache_world_size=None):
    """Shapes and derived scalars of DirectMPIGO.__init__ (lib/dmpigo.py:19-154)."""
    st = {'kind': 'dmpigo'}
    st['xyz_min'] = torch.Tensor(xyz_min)
    st['xyz_max'] = torch.Tensor(xyz_max)
    st['fast_color_thres'] = fast_color_thres
    st['mpi_depth'] = mpi_depth
    # lib/dmpigo.py:160-164
    r = (num_voxels / mpi_depth / (st['xyz_max'] - st['xyz_min'])[:2].prod()).sqrt()
    ws = torch.zeros(3, dtype=torch.long)
    ws[:2] = (st['xyz_max'] - st['xyz_min'])[:2] * r
    ws[2] = mpi_depth
    st['world_size'] = ws
    st['voxel_size_ratio'] = 256. / mpi_depth
    wsl = ws.tolist()
    st['density'] = torch.zeros([1, 1, *wsl])
    # lib/dmpigo.py:48-58: depth-dependent bias grid [1,1,1,1,D]
    act = torch.zeros([1, 1, 1, 1, mpi_depth])
    g = np.full([mpi_depth], 1. / mpi_depth - 1e-6)
    p = [1 - g[0]]
    for i in range(1, len(g)):
        p.append((1 - g[:i + 1].sum()) / (1 - g[:i].sum()))
    for i in range(len(p)):
        act[..., i].fill_(np.log(p[i] ** (-1 / st['voxel_size_ratio']) - 1))
    st['act_shift_grid'] = act
    st['rgbnet_dim'] = rgbnet_dim
    if rgbnet_dim <= 0:
        st['k0_dim'] = 3
        st['rgbnet'] = None
    else:
        st['k0_dim'] = rgbnet_dim
        st['viewfreq'] = torch.FloatTensor([(2 ** i) for i in range(viewbase_pe)])
        st['posfreq'] = torch.FloatTensor([(2 ** i) for i in range(spatial_pe)])
        st['dim0'] = (3 + 3 * viewbase_pe * 2 + 3 + 3 * spatial_pe * 2) + st['k0_dim']
        dims = [st['dim0']] + [rgbnet_width] * (rgbnet_depth - 1) + [3]
        st['rgbnet'] = [(torch.zeros(dims[i + 1], dims[i]), torch.zeros(dims[i + 1])) for i in range(len(dims) - 1)]
    st['k0'] = torch.zeros([1, st['k0_dim'], *wsl])
    if mask_cache_world_size is None:
        mask_cache_world_size = wsl
    st['mask_cache'] = mask_grid_state(torch.ones(list(mask_cache_world_size), dtype=torch.bool),
                                       st['xyz_min'], st['xyz_max'])
    return st


def dcvgo_state(xyz_min, xyz_max, num_voxels, num_voxels_base, alpha_init, fast_color_thres, bg_len=0.2,
                rgbnet_dim=0, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4, mask_cache_world_size=None):
    """Shapes and derived scalars of DirectContractedVoxGO.__init__ (lib/dcvgo.py:28-128)."""
    st = {'kind': 'dcvgo', 'bg_len': bg_len}
    xyz_min = torch.Tensor(xyz_min)
    xyz_max = torch.Tensor(xyz_max)
    st['scene_center'] = (xyz_min + xyz_max) * 0.5
    st['scene_radius'] = (xyz_max - xyz_min) * 0.5
    st['xyz_min'] = torch.Tensor([-1, -1, -1]) - bg_len
    st['xyz_max'] = torch.Tensor([1, 1, 1]) + bg_len
    st['fast_color_thres'] = fast_color_thres
    st['voxel_size_base'] = ((st['xyz_max'] - st['xyz_min']).prod() / num_voxels_base).pow(1 / 3)
    st['voxel_size'] = ((st['xyz_max'] - st['xyz_min']).prod() / num_voxels).pow(1 / 3)
    st['world_size'] = ((st['xyz_max'] - st['xyz_min']) / st['voxel_size']).long()
    st['world_len'] = st['world_size'][0].item()
    st['voxel_size_ratio'] = st['voxel_size'] / st['voxel_size_base']
    st['act_shift'] = torch.FloatTensor([np.log(1 / (1 - alpha_init) - 1)])
    ws = st['world_size'].tolist()
    st['density'] = torch.zeros([1, 1, *ws])
    st['rgbnet_dim'] = rgbnet_dim
    if rgbnet_dim <= 0:
        st['k0_dim'] = 3
        st['rgbnet'] = None
    else:
        st['k0_dim'] = rgbnet_dim
        st['viewfreq'] = torch.FloatTensor([(2 ** i) for i in range(viewbase_pe)])
        dim0 = 3 + 3 * viewbase_pe * 2 + rgbnet_dim
        st['dim0'] = dim0
        dims = [dim0] + [rgbnet_width] * (rgbnet_depth - 1) + [3]
        st['rgbnet'] = [(torch.zeros(dims[i + 1], dims[i]), torch.zeros(dims[i + 1])) for i in range(len(dims) - 1)]
    st['k0'] = torch.zeros([1, st['k0_dim'], *ws])
    if mask_cache_world_size is None:
        mask_cache_world_size = ws
    st['mask_cache'] = mask_grid_state(torch.ones(list(mask_cache_world_size), dtype=torch.bool), st['xyz_min'], st['xyz_max'])
    return st


def state_to(st, device):
    out = {}
    for k, v in st.items():
        if torch.is_tensor(v):
            out[k] = v.to(device)
        elif isinstance(v, dict):
            out[k] = state_to(v, device)
        elif isinstance(v, list) and v and isinstance(v[0], tuple):
            out[k] = [tuple(t.to(device) for t in pair) for pair in v]
        else:
            out[k] = v
    return out


# ----------------------------------------------------------------------------------------------
# grid primitives
# ----------------------------------------------------------------------------------------------
def dense_grid(grid, xyz, xyz_min, xyz_max):
    """DenseGrid.forward, lib/grid.py:117-128 (normalise, flip, trilinear align_corners=True)."""
    channels = grid.shape[1]
    shape = xyz.shape[:-1]
    xyz = xyz.reshape(1, 1, 1, -1, 3)
    ind_norm = ((xyz - xyz_min) / (xyz_max - xyz_min)).flip((-1,)) * 2 - 1
    out = F.grid_sample(grid, ind_norm, mode='bilinear', align_corners=True)
    out = out.reshape(channels, -1).T.reshape(*shape, channels)
    if channels == 1:
        out = out.squeeze(-1)
    return out


def mask_grid(mc, xyz, ops):
    """MaskGrid.forward, lib/grid.py:295-304."""
    shape = xyz.shape[:-1]
    xyz = xyz.reshape(-1, 3)
    mask = ops.maskcache_lookup(mc['mask'], xyz.contiguous(), mc['xyz2ijk_scale'], mc['xyz2ijk_shift'])
    return mask.reshape(shape)


def mlp(layers, x):
    """nn.Sequential(Linear, ReLU, ..., Linear), lib/dvgo.py:116-123."""
    for i, (w, b) in enumerate(layers):
        x = F.linear(x, w, b)
        if i + 1 < len(layers):
            x = F.relu(x)
    return x


def _segment_sum(src, index, out):
    """torch_scatter.segment_coo(src, index, out, reduce='sum') for a sorted index."""
    return out.index_add_(0, index, src)


def _early_out_counts(ids_m, ids_d, ids_a, i_end, alphainv_last, N):
    """Per-ray sample counts with the transmittance early-out applied.

    The reference materialises every in-box sample before it knows where a ray saturates
    (render_utils_kernel.cu:597 only zeroes the later weights), so its mask lookups / density fetches
    cover ALL in-box samples (`S_m_all`, `S_d_all`).  A marcher that stops at the early-out never
    visits the samples behind it; SURVEY.md section 8(d) defines the roofline counts on those visited
    samples.  Returns int64 [N,2]: in-box samples and occupancy hits with step <= the step of the
    last composited sample of the ray (all of them for rays that never reached T < 1e-3)."""
    ray_a, step_a = ids_a
    dev = alphainv_last.device
    big = torch.iinfo(torch.int64).max
    last_step = torch.full((N,), big, dtype=torch.int64, device=dev)
    if ray_a.numel():
        term = (alphainv_last.double() < 1e-3) & (i_end > 0)
        idx = (i_end - 1).clamp(min=0)
        last_step = torch.where(term, step_a[idx.clamp(max=ray_a.numel() - 1)], last_step)
    out = torch.zeros((N, 2), dtype=torch.int64, device=dev)
    for col, (rid, sid) in enumerate((ids_m, ids_d)):
        keep = sid <= last_step[rid]
        out[:, col] = torch.zeros(N, dtype=torch.int64, device=dev).index_add_(0, rid[keep], torch.ones_like(rid[keep]))
    return out


def _trace(trace, ray_id, weights, rgb_feat, diffuse, step_id, s):
    """Record the shaded samples of a forward pass: ray_id [S], weights [S], the rgbnet's inputs rgb_feat [S, dim0] (the
    k0 colour logits [S, 3] for a model without an rgbnet) and, for rgbnet_direct=False, the diffuse logits [S, 3] added
    before the sigmoid (else None); step_id [S] and the depth coordinate s [S] of each."""
    if trace is not None:
        trace.update(ray_id=ray_id.clone(), weights=weights.clone(), rgb_feat=rgb_feat.clone(),
                     diffuse=None if diffuse is None else diffuse.clone(), step_id=step_id.clone(), s=s.clone())


def _trace_occupied(trace, ray_id, step_id, pts, density, alpha):
    """Record every occupied sample (the mask lookup hit it), in ray and step order: its ray, step, position, density as
    it enters raw2alpha (before the shift) and alpha."""
    if trace is not None:
        trace['occupied'] = dict(ray_id=ray_id.clone(), step_id=step_id.clone(), pts=pts.clone(),
                                 density=density.flatten().clone(), alpha=alpha.flatten().clone())


def _trace_composited(trace, ray_id, step_id, alpha, T, i_end):
    """Record the samples alpha2weight composites (the alpha threshold's survivors, or every occupied sample without a
    threshold): ray, step, alpha and the transmittance T in front of the sample; and per ray i_end, one past the last
    sample it composited before the T < 1e-3 early-out."""
    if trace is not None:
        trace['composited'] = dict(ray_id=ray_id.clone(), step_id=step_id.clone(), alpha=alpha.clone(), T=T.clone(),
                                   i_end=i_end.clone())


def _add_stats(stats, ids_m, ids_d, S_c, ray_stats, ray_id_c, N):
    """S_m/S_d: visited before the early-out (what a fused marcher touches); *_all: what the
    reference's unfused pipeline touches; S_c: samples shaded (identical in both)."""
    stats['S_m'] = stats.get('S_m', 0) + int(ray_stats[:, 0].sum())
    stats['S_d'] = stats.get('S_d', 0) + int(ray_stats[:, 1].sum())
    stats['S_c'] = stats.get('S_c', 0) + S_c
    stats['S_m_all'] = stats.get('S_m_all', 0) + ids_m[0].shape[0]
    stats['S_d_all'] = stats.get('S_d_all', 0) + ids_d[0].shape[0]
    stats['n_rays'] = stats.get('n_rays', 0) + N


# ----------------------------------------------------------------------------------------------
# forward passes
# ----------------------------------------------------------------------------------------------
@torch.no_grad()
def dvgo_forward(st, rays_o, rays_d, viewdirs, ops, stats=None, trace=None, **render_kwargs):
    """DirectVoxGO.forward (lib/dvgo.py:327-448) at inference (global_step=None)."""
    dev = rays_o.device
    N = len(rays_o)
    # sample_ray, lib/dvgo.py:307-325
    far = 1e9
    stepdist = render_kwargs['stepsize'] * st['voxel_size']
    N_samples = int((st['max_world_size'] - 1) / render_kwargs['stepsize']) + 1
    ray_pts, mask_outbbox, ray_id, step_id, N_steps, t_min, t_max = ops.sample_pts_on_rays(
        rays_o.contiguous(), rays_d.contiguous(), st['xyz_min'], st['xyz_max'],
        render_kwargs['near'], far, float(stepdist))
    mask_inbbox = ~mask_outbbox
    ray_pts = ray_pts[mask_inbbox]
    ray_id = ray_id[mask_inbbox]
    step_id = step_id[mask_inbbox]
    interval = float(render_kwargs['stepsize'] * st['voxel_size_ratio'])
    ids_m = (ray_id, step_id)

    mask1 = mask_grid(st['mask_cache'], ray_pts, ops)
    ray_pts = ray_pts[mask1]
    ray_id = ray_id[mask1]
    step_id = step_id[mask1]
    ids_d = (ray_id, step_id)

    density = dense_grid(st['density'], ray_pts, st['xyz_min'], st['xyz_max'])
    alpha = ops.raw2alpha(density.flatten().contiguous(), float(st['act_shift']), interval)[1].reshape(density.shape)
    _trace_occupied(trace, ray_id, step_id, ray_pts, density, alpha)
    if st['fast_color_thres'] > 0:
        mask2 = (alpha > st['fast_color_thres'])
        ray_pts = ray_pts[mask2]
        ray_id = ray_id[mask2]
        step_id = step_id[mask2]
        alpha = alpha[mask2]

    weights, T_in, alphainv_last, _, i_end = ops.alpha2weight(alpha.contiguous(), ray_id.contiguous(), N)
    _trace_composited(trace, ray_id, step_id, alpha, T_in, i_end)
    ray_stats = _early_out_counts(ids_m, ids_d, (ray_id, step_id), i_end, alphainv_last, N) if stats is not None else None
    if st['fast_color_thres'] > 0:
        mask3 = (weights > st['fast_color_thres'])
        weights = weights[mask3]
        alpha = alpha[mask3]
        ray_pts = ray_pts[mask3]
        ray_id = ray_id[mask3]
        step_id = step_id[mask3]
    S_c = ray_pts.shape[0]
    s = (step_id + 0.5) / N_samples

    k0 = dense_grid(st['k0'], ray_pts, st['xyz_min'], st['xyz_max'])
    if st['rgbnet'] is None:
        _trace(trace, ray_id, weights, k0, None, step_id, s)
        rgb_raw = torch.sigmoid(k0)
    else:
        if st['rgbnet_direct']:
            k0_view = k0
        else:
            k0_view = k0[:, 3:]
            k0_diffuse = k0[:, :3]
        viewdirs_emb = (viewdirs.unsqueeze(-1) * st['viewfreq']).flatten(-2)
        viewdirs_emb = torch.cat([viewdirs, viewdirs_emb.sin(), viewdirs_emb.cos()], -1)
        viewdirs_emb = viewdirs_emb.flatten(0, -2)[ray_id]
        rgb_feat = torch.cat([k0_view, viewdirs_emb], -1)
        _trace(trace, ray_id, weights, rgb_feat, None if st['rgbnet_direct'] else k0_diffuse, step_id, s)
        rgb_logit = mlp(st['rgbnet'], rgb_feat)
        if st['rgbnet_direct']:
            rgb_raw = torch.sigmoid(rgb_logit)
        else:
            rgb_raw = torch.sigmoid(rgb_logit + k0_diffuse)

    rgb_feature = _segment_sum(weights.unsqueeze(-1) * rgb_raw, ray_id, torch.zeros([N, 3], device=dev))
    rgb_marched = rgb_feature                      # alias, lib/dvgo.py:425
    rgb_marched += (alphainv_last.unsqueeze(-1) * render_kwargs['bg'])
    ret = {
        'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched,
        'rgb_feature': rgb_feature, 'raw_alpha': alpha, 'raw_rgb': rgb_raw, 'ray_id': ray_id,
    }
    if render_kwargs.get('render_depth', False):
        ret['depth'] = _segment_sum(weights * s, ray_id, torch.zeros([N], device=dev))
    if stats is not None:
        _add_stats(stats, ids_m, ids_d, S_c, ray_stats, ray_id, N)
        ret['_ray_stats'] = ray_stats
        ret['_N_steps'] = N_steps
        ret['_t_min'] = t_min
        ret['_t_max'] = t_max
        ret['_step_id'] = step_id
    return ret


@torch.no_grad()
def dmpigo_forward(st, rays_o, rays_d, viewdirs, ops, stats=None, trace=None, **render_kwargs):
    """DirectMPIGO.forward (lib/dmpigo.py:292-427) at inference (global_step=None)."""
    dev = rays_o.device
    N = len(rays_o)
    assert render_kwargs['near'] == 0 and render_kwargs['far'] == 1
    # sample_ray, lib/dmpigo.py:276-290
    N_samples = int((st['mpi_depth'] - 1) / render_kwargs['stepsize']) + 1
    ray_pts, mask_outbbox = ops.sample_ndc_pts_on_rays(
        rays_o.contiguous(), rays_d.contiguous(), st['xyz_min'], st['xyz_max'], N_samples)
    mask_inbbox = ~mask_outbbox
    ray_pts = ray_pts.view(-1, 3)
    ray_pts = ray_pts[mask_inbbox.view(-1)]
    ray_id = torch.arange(mask_inbbox.shape[0], device=dev).view(-1, 1).expand_as(mask_inbbox)[mask_inbbox]
    step_id = torch.arange(mask_inbbox.shape[1], device=dev).view(1, -1).expand_as(mask_inbbox)[mask_inbbox]
    interval = float(render_kwargs['stepsize'] * st['voxel_size_ratio'])
    ids_m = (ray_id, step_id)

    mask1 = mask_grid(st['mask_cache'], ray_pts, ops)
    ray_pts = ray_pts[mask1]
    ray_id = ray_id[mask1]
    step_id = step_id[mask1]
    ids_d = (ray_id, step_id)

    density = dense_grid(st['density'], ray_pts, st['xyz_min'], st['xyz_max']) + \
        dense_grid(st['act_shift_grid'], ray_pts, st['xyz_min'], st['xyz_max'])
    alpha = ops.raw2alpha(density.flatten().contiguous(), 0, interval)[1].reshape(density.shape)
    _trace_occupied(trace, ray_id, step_id, ray_pts, density, alpha)
    if st['fast_color_thres'] > 0:
        mask2 = (alpha > st['fast_color_thres'])
        ray_pts = ray_pts[mask2]
        ray_id = ray_id[mask2]
        step_id = step_id[mask2]
        alpha = alpha[mask2]

    weights, T_in, alphainv_last, _, i_end = ops.alpha2weight(alpha.contiguous(), ray_id.contiguous(), N)
    _trace_composited(trace, ray_id, step_id, alpha, T_in, i_end)
    ray_stats = _early_out_counts(ids_m, ids_d, (ray_id, step_id), i_end, alphainv_last, N) if stats is not None else None
    if st['fast_color_thres'] > 0:
        mask3 = (weights > st['fast_color_thres'])
        ray_pts = ray_pts[mask3]
        ray_id = ray_id[mask3]
        step_id = step_id[mask3]
        alpha = alpha[mask3]
        weights = weights[mask3]
    S_c = ray_pts.shape[0]
    s = (step_id + 0.5) / N_samples

    vox_emb = dense_grid(st['k0'], ray_pts, st['xyz_min'], st['xyz_max'])
    pe_spa = ((ray_pts - st['xyz_min']) / (st['xyz_max'] - st['xyz_min'])).flip((-1,)) * 2 - 1
    if st['rgbnet'] is None:
        _trace(trace, ray_id, weights, vox_emb, None, step_id, s)
        rgb_raw = torch.sigmoid(vox_emb)
    else:
        viewdirs_emb = (viewdirs.unsqueeze(-1) * st['viewfreq']).flatten(-2)
        viewdirs_emb = torch.cat([viewdirs, viewdirs_emb.sin(), viewdirs_emb.cos()], -1)
        viewdirs_emb = viewdirs_emb[ray_id]
        pe_emb = (pe_spa.unsqueeze(-1) * st['posfreq']).flatten(-2)
        pe_emb = torch.cat([pe_spa, pe_emb.sin(), pe_emb.cos()], -1)
        rgb_feat = torch.cat([vox_emb, pe_emb, viewdirs_emb], -1)
        _trace(trace, ray_id, weights, rgb_feat, None, step_id, s)
        rgb_logit = mlp(st['rgbnet'], rgb_feat)
        rgb_raw = torch.sigmoid(rgb_logit)

    rgb_feature = _segment_sum(weights.unsqueeze(-1) * rgb_raw, ray_id, torch.zeros([N, 3], device=dev))
    rgb_marched = rgb_feature                      # alias, lib/dmpigo.py:392
    rgb_marched += (alphainv_last.unsqueeze(-1) * render_kwargs['bg'])   # global_step is None branch, :397
    ret = {
        'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched,
        'rgb_feature': rgb_feature, 'raw_alpha': alpha, 'raw_rgb': rgb_raw, 'ray_id': ray_id,
        'n_max': N_samples, 's': s,
    }
    if render_kwargs.get('render_depth', False):
        ret['depth'] = _segment_sum(weights * s, ray_id, torch.zeros([N], device=dev))
    if stats is not None:
        _add_stats(stats, ids_m, ids_d, S_c, ray_stats, ray_id, N)
        ret['_ray_stats'] = ray_stats
        ret['_step_id'] = step_id
    return ret


@torch.no_grad()
def dcvgo_forward(st, rays_o, rays_d, viewdirs, ops, stats=None, trace=None, **render_kwargs):
    """DirectContractedVoxGO.forward (lib/dcvgo.py:264-382, sample_ray :226-262) at inference."""
    dev = rays_o.device
    N = len(rays_o)
    stepsize = render_kwargs['stepsize']
    # sample_ray
    o = (rays_o - st['scene_center']) / st['scene_radius']
    d = rays_d / rays_d.norm(dim=-1, keepdim=True)
    N_inner = int(2 / (2 + 2 * st['bg_len']) * st['world_len'] / stepsize) + 1
    N_outer = N_inner
    b_inner = torch.linspace(0, 2, N_inner + 1, device=dev)
    b_outer = 2 / torch.linspace(1, 1 / 128, N_outer + 1, device=dev)
    t = torch.cat([(b_inner[1:] + b_inner[:-1]) * 0.5, (b_outer[1:] + b_outer[:-1]) * 0.5])
    ray_pts = o[:, None, :] + d[:, None, :] * t[None, :, None]
    norm = ray_pts.abs().amax(dim=-1, keepdim=True)
    inner_mask = (norm <= 1)
    ray_pts = torch.where(inner_mask, ray_pts, ray_pts / norm * ((1 + st['bg_len']) - st['bg_len'] / norm))
    inner_mask = inner_mask.squeeze(-1)
    n_max = len(t)
    interval = float(stepsize * st['voxel_size_ratio'])
    ray_id = torch.arange(N, device=dev).view(-1, 1).expand(N, n_max).flatten()
    step_id = torch.arange(n_max, device=dev).view(1, -1).expand(N, n_max).flatten()
    # skip oversampled points outside the scene bbox
    mask = inner_mask.clone()
    dist_thres = (2 + 2 * st['bg_len']) / st['world_len'] * stepsize * 0.95
    dist = (ray_pts[:, 1:] - ray_pts[:, :-1]).norm(dim=-1)
    mask[:, 1:] |= ops.cumdist_thres(dist.contiguous(), dist_thres)
    ray_pts = ray_pts[mask]
    tt = t[None].repeat(N, 1)[mask]
    ray_id = ray_id[mask.flatten()]
    step_id = step_id[mask.flatten()]
    ids_m = (ray_id, step_id)

    m1 = mask_grid(st['mask_cache'], ray_pts, ops)
    ray_pts, tt, ray_id, step_id = ray_pts[m1], tt[m1], ray_id[m1], step_id[m1]
    ids_d = (ray_id, step_id)

    density = dense_grid(st['density'], ray_pts, st['xyz_min'], st['xyz_max'])
    alpha = ops.raw2alpha(density.flatten().contiguous(), float(st['act_shift']), interval)[1].reshape(density.shape)
    _trace_occupied(trace, ray_id, step_id, ray_pts, density, alpha)
    if st['fast_color_thres'] > 0:
        m2 = (alpha > st['fast_color_thres'])
        ray_pts, tt, ray_id, step_id, alpha = ray_pts[m2], tt[m2], ray_id[m2], step_id[m2], alpha[m2]
    weights, T_in, alphainv_last, _, i_end = ops.alpha2weight(alpha.contiguous(), ray_id.contiguous(), N)
    _trace_composited(trace, ray_id, step_id, alpha, T_in, i_end)
    ray_stats = _early_out_counts(ids_m, ids_d, (ray_id, step_id), i_end, alphainv_last, N) if stats is not None else None
    if st['fast_color_thres'] > 0:
        m3 = (weights > st['fast_color_thres'])
        ray_pts, tt, ray_id, step_id, alpha, weights = ray_pts[m3], tt[m3], ray_id[m3], step_id[m3], alpha[m3], weights[m3]
    S_c = ray_pts.shape[0]
    s = 1 - 1 / (1 + tt)

    k0 = dense_grid(st['k0'], ray_pts, st['xyz_min'], st['xyz_max'])
    if st['rgbnet'] is None:
        _trace(trace, ray_id, weights, k0, None, step_id, s)
        rgb = torch.sigmoid(k0)
    else:
        viewdirs_emb = (viewdirs.unsqueeze(-1) * st['viewfreq']).flatten(-2)
        viewdirs_emb = torch.cat([viewdirs, viewdirs_emb.sin(), viewdirs_emb.cos()], -1)
        viewdirs_emb = viewdirs_emb.flatten(0, -2)[ray_id]
        rgb_feat = torch.cat([k0, viewdirs_emb], -1)
        _trace(trace, ray_id, weights, rgb_feat, None, step_id, s)
        rgb = torch.sigmoid(mlp(st['rgbnet'], rgb_feat))
    rgb_marched = _segment_sum(weights.unsqueeze(-1) * rgb, ray_id, torch.zeros([N, 3], device=dev))
    rgb_marched += (alphainv_last.unsqueeze(-1) * render_kwargs['bg'])
    ret = {'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched, 'rgb_feature': rgb_marched,
           'raw_alpha': alpha, 'raw_rgb': rgb, 'ray_id': ray_id, 'step_id': step_id, 'n_max': n_max, 't': tt, 's': s}
    if render_kwargs.get('render_depth', False):
        ret['depth'] = _segment_sum(weights * s, ray_id, torch.zeros([N], device=dev))
    if stats is not None:
        _add_stats(stats, ids_m, ids_d, S_c, ray_stats, ray_id, N)
        ret['_ray_stats'] = ray_stats
    return ret


def forward(st, rays_o, rays_d, viewdirs, ops, stats=None, trace=None, **render_kwargs):
    """trace: optional dict that receives the shaded samples (see _trace), and under 'occupied' / 'composited' the
    samples that hit the occupancy mask and those alpha2weight composited (_trace_occupied / _trace_composited)."""
    if st['kind'] == 'dcvgo':
        return dcvgo_forward(st, rays_o, rays_d, viewdirs, ops, stats=stats, trace=trace, **render_kwargs)
    fn = dvgo_forward if st['kind'] == 'dvgo' else dmpigo_forward
    return fn(st, rays_o, rays_d, viewdirs, ops, stats=stats, trace=trace, **render_kwargs)


@torch.no_grad()
def render_rays_chunked(st, rays_o, rays_d, viewdirs, ops, chunk=8192, stats=None, **render_kwargs):
    """The chunk loop of render_viewpoints (run_sr.py:121-128): 8192-ray chunks, concatenated."""
    keys = ['rgb_marched', 'depth', 'alphainv_last', 'rgb_feature']
    outs = []
    for ro, rd, vd in zip(rays_o.split(chunk, 0), rays_d.split(chunk, 0), viewdirs.split(chunk, 0)):
        r = forward(st, ro, rd, vd, ops, stats=stats, **render_kwargs)
        outs.append({k: v for k, v in r.items() if k in keys})
    return {k: torch.cat([o[k] for o in outs]) for k in outs[0].keys()}


# ----------------------------------------------------------------------------------------------
# rays (lib/dvgo.py:516-582)
# ----------------------------------------------------------------------------------------------
def get_rays(H, W, K, c2w, inverse_y, flip_x, flip_y, mode='center'):
    """get_rays, lib/dvgo.py:516-544."""
    i, j = torch.meshgrid(
        torch.linspace(0, W - 1, W, device=c2w.device),
        torch.linspace(0, H - 1, H, device=c2w.device), indexing='ij')
    i = i.t().float()
    j = j.t().float()
    if mode == 'center':
        i, j = i + 0.5, j + 0.5
    elif mode != 'lefttop':
        raise NotImplementedError
    if flip_x:
        i = i.flip((1,))
    if flip_y:
        j = j.flip((0,))
    if inverse_y:
        dirs = torch.stack([(i - K[0][2]) / K[0][0], (j - K[1][2]) / K[1][1], torch.ones_like(i)], -1)
    else:
        dirs = torch.stack([(i - K[0][2]) / K[0][0], -(j - K[1][2]) / K[1][1], -torch.ones_like(i)], -1)
    rays_d = torch.sum(dirs[..., np.newaxis, :] * c2w[:3, :3], -1)
    rays_o = c2w[:3, 3].expand(rays_d.shape)
    return rays_o, rays_d


def ndc_rays(H, W, focal, near, rays_o, rays_d):
    """ndc_rays, lib/dvgo.py:557-574."""
    t = -(near + rays_o[..., 2]) / rays_d[..., 2]
    rays_o = rays_o + t[..., None] * rays_d
    o0 = -1. / (W / (2. * focal)) * rays_o[..., 0] / rays_o[..., 2]
    o1 = -1. / (H / (2. * focal)) * rays_o[..., 1] / rays_o[..., 2]
    o2 = 1. + 2. * near / rays_o[..., 2]
    d0 = -1. / (W / (2. * focal)) * (rays_d[..., 0] / rays_d[..., 2] - rays_o[..., 0] / rays_o[..., 2])
    d1 = -1. / (H / (2. * focal)) * (rays_d[..., 1] / rays_d[..., 2] - rays_o[..., 1] / rays_o[..., 2])
    d2 = -2. * near / rays_o[..., 2]
    return torch.stack([o0, o1, o2], -1), torch.stack([d0, d1, d2], -1)


def get_rays_of_a_view(H, W, K, c2w, ndc, inverse_y, flip_x, flip_y, mode='center'):
    """get_rays_of_a_view, lib/dvgo.py:577-582 (viewdirs normalised BEFORE the NDC warp)."""
    rays_o, rays_d = get_rays(H, W, K, c2w, inverse_y=inverse_y, flip_x=flip_x, flip_y=flip_y, mode=mode)
    viewdirs = rays_d / rays_d.norm(dim=-1, keepdim=True)
    if ndc:
        rays_o, rays_d = ndc_rays(H, W, K[0][0], 1., rays_o, rays_d)
    return rays_o, rays_d, viewdirs


def psnr(a, b):
    """-10 log10 mse, as lib/utils.py:18 mse2psnr; +inf for identical inputs."""
    mse = torch.mean((a.double() - b.double()) ** 2).item()
    return float('inf') if mse == 0 else -10. * math.log10(mse)
