"""Float64 restatement of the three training forwards (DirectVoxGO, DirectMPIGO, DirectContractedVoxGO) with plain
autograd, the composite loss of the reference's training loop, and the error bounds the GPU gradient tests hold the
library to.  Helpers only; the error model is written down in test_gpu_train_grad.py's module docstring.

The restatement follows lib/dvgo.py:327-448, lib/dmpigo.py:292-427 and lib/dcvgo.py:262-382.  Sample positions and
occupancy are the fp32 values of the oracle's CPU ops (oracle.ops.CpuOps: sample_pts_on_rays, sample_ndc_pts_on_rays,
maskcache_lookup, cumdist_thres), which other tests pin bit-exact to the reference's kernels: the reference
differentiates at those fp32 points.  Everything after them is fp64: trilinear lookup by F.grid_sample on fp64 copies
of the grids, the alpha formula, the transmittance scan with the T < 1e-3 early stop, both fast_color_thres
compactions, the rgbnet on fp64 copies of its weights, and index_add segment sums.  No custom autograd Function.

Where fp32 and fp64 could disagree on a sample's fate (alpha > thres, weights > thres, T < 1e-3, cumdist > thres; and
alphainv_last at the entropy loss's clamp) the
relative distance to the threshold, |q - thres| / |q|, is recorded per candidate sample, so that a test can assert it
against the relative error of q and report a borderline sample as such.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.ops import CpuOps

U = 2.0 ** -24
A_GAUSS = 0.05
T_STOP = 1e-3                       # render_utils_kernel.cu:597


# ---------------------------------------------------------------------------------------------------------------------
# parameters: a plain dict of fp64 leaves (grids, rgbnet) and fp32 constants, from a k4nerf model or an oracle state
# ---------------------------------------------------------------------------------------------------------------------
def _leaf(t):
    return t.detach().to('cpu', torch.float64).clone().requires_grad_(True)


def params_from_model(m):
    """fp64 copies of a k4nerf model's trainable tensors and its fp32 constants."""
    from k4nerf import _lib
    from k4nerf._scene import linear_layers
    kind = {_lib.K4_KIND_DVGO: 'dvgo', _lib.K4_KIND_DMPIGO: 'dmpigo', _lib.K4_KIND_DCVGO: 'dcvgo'}[m._k4_kind]
    cpu = lambda t: t.detach().cpu() if torch.is_tensor(t) else t
    P = dict(kind=kind, xyz_min=cpu(m.xyz_min).float(), xyz_max=cpu(m.xyz_max).float(),
             density=_leaf(m.density.grid), k0=_leaf(m.k0.grid), fast_color_thres=float(m.fast_color_thres),
             mask=cpu(m.mask_cache.mask), mask_scale=cpu(m.mask_cache.xyz2ijk_scale), mask_shift=cpu(m.mask_cache.xyz2ijk_shift),
             voxel_size_ratio=cpu(m.voxel_size_ratio), act=getattr(m, 'act_type', 'relu'),
             rgbnet_direct=bool(getattr(m, 'rgbnet_direct', True)))
    if P['act'] not in ('relu', 'gauss', 'lkrelu'):
        P['act'] = 'relu'
    if kind == 'dvgo':
        P.update(voxel_size=cpu(m.voxel_size), max_world_size=int(m.max_world_size), act_shift=float(m.act_shift))
    elif kind == 'dmpigo':
        P.update(mpi_depth=int(m.mpi_depth), act_shift_grid=cpu(m.act_shift.grid).double())
    else:
        P.update(act_shift=float(m.act_shift), scene_center=cpu(m.scene_center).float(),
                 scene_radius=cpu(m.scene_radius).float(), bg_len=float(m.bg_len), world_len=int(m.world_len))
    P['rgbnet'] = None
    if m.rgbnet is not None:
        P['rgbnet'] = [(_leaf(l.weight), _leaf(l.bias)) for l in linear_layers(m.rgbnet)]
        P['viewfreq'] = cpu(m.viewfreq).float()
        if kind == 'dmpigo':
            P['posfreq'] = cpu(m.posfreq).float()
            if P['act'] == 'gauss':
                P['gauss_a'] = float(m.rgbnet[1].a)
    return P


def params_from_state(st, act='relu'):
    """The same dict from an oracle scene state (oracle/pipeline.py)."""
    kind = st['kind']
    mc = st['mask_cache']
    P = dict(kind=kind, xyz_min=st['xyz_min'].float(), xyz_max=st['xyz_max'].float(), density=_leaf(st['density']),
             k0=_leaf(st['k0']), fast_color_thres=float(st['fast_color_thres']), mask=mc['mask'],
             mask_scale=mc['xyz2ijk_scale'], mask_shift=mc['xyz2ijk_shift'], voxel_size_ratio=st['voxel_size_ratio'],
             act=act, rgbnet_direct=bool(st.get('rgbnet_direct', True)))
    if kind == 'dvgo':
        P.update(voxel_size=st['voxel_size'], max_world_size=int(st['max_world_size']), act_shift=float(st['act_shift']))
    elif kind == 'dmpigo':
        P.update(mpi_depth=int(st['mpi_depth']), act_shift_grid=st['act_shift_grid'].double())
    else:
        P.update(act_shift=float(st['act_shift']), scene_center=st['scene_center'].float(),
                 scene_radius=st['scene_radius'].float(), bg_len=float(st['bg_len']), world_len=int(st['world_len']))
    P['rgbnet'] = None
    if st['rgbnet'] is not None:
        P['rgbnet'] = [(_leaf(w), _leaf(b)) for w, b in st['rgbnet']]
        P['viewfreq'] = st['viewfreq'].float()
        if kind == 'dmpigo':
            P['posfreq'] = st['posfreq'].float()
            P['gauss_a'] = A_GAUSS
    return P


def trainable(P):
    """name -> fp64 leaf, with the k4nerf parameter names."""
    out = {'density.grid': P['density'], 'k0.grid': P['k0']}
    for i, (w, b) in enumerate(P['rgbnet'] or []):
        out[f'rgbnet.L{i}.weight'], out[f'rgbnet.L{i}.bias'] = w, b
    return out


# ---------------------------------------------------------------------------------------------------------------------
# fp64 building blocks
# ---------------------------------------------------------------------------------------------------------------------
def grid_lookup(grid, pts, lo, hi):
    """DenseGrid.forward (lib/grid.py:117-128) in fp64 on fp32 points: [S, C]."""
    C = grid.shape[1]
    xyz = pts.double().reshape(1, 1, 1, -1, 3)
    ind = ((xyz - lo.double()) / (hi.double() - lo.double())).flip((-1,)) * 2 - 1
    return F.grid_sample(grid, ind, mode='bilinear', align_corners=True).reshape(C, -1).T


def corners(pts, lo, hi, shape):
    """The 8 trilinear corners of each point: flat voxel index [S, 8] (-1 outside the grid) and weight [S, 8], fp64."""
    X, Y, Z = shape
    c = (pts.double() - lo.double()) / (hi.double() - lo.double()) * (torch.tensor([X, Y, Z], dtype=torch.float64) - 1)
    f = c.floor()
    fr = c - f
    f = f.long()
    idx, w = [], []
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                i, j, k = f[:, 0] + dx, f[:, 1] + dy, f[:, 2] + dz
                ok = (i >= 0) & (i < X) & (j >= 0) & (j < Y) & (k >= 0) & (k < Z)
                wt = ((fr[:, 0] if dx else 1 - fr[:, 0]) * (fr[:, 1] if dy else 1 - fr[:, 1]) *
                      (fr[:, 2] if dz else 1 - fr[:, 2]))
                idx.append(torch.where(ok, (i * Y + j) * Z + k, torch.full_like(i, -1)))
                w.append(torch.where(ok, wt, torch.zeros_like(wt)))
    return torch.stack(idx, 1), torch.stack(w, 1)


def scatter_corners(vals, idx, nvox):
    """sum over samples and corners of vals [S, 8] into a flat [nvox] fp64 grid (out-of-grid corners dropped)."""
    out = torch.zeros(nvox, dtype=torch.float64)
    ok = idx >= 0
    return out.index_add_(0, idx[ok], vals[ok].double())


def act_fn(x, act, a=A_GAUSS):
    if act == 'relu':
        return F.relu(x)
    if act == 'gauss':
        a32 = float(np.float32(a))                       # GaussianActivation holds a as an fp32 parameter
        return torch.exp(-x ** 2 / (2 * a32 ** 2))
    return F.leaky_relu(x, float(np.float32(0.01)))


def _segments(ray_id, n):
    """position of every sample within its ray, and the longest ray (ray_id sorted)."""
    counts = torch.bincount(ray_id, minlength=n) if ray_id.numel() else torch.zeros(n, dtype=torch.long)
    start = torch.cumsum(counts, 0) - counts
    pos = torch.arange(ray_id.numel()) - start[ray_id]
    return pos, int(counts.max()) if n else 0, counts


def _dense(v, ray_id, pos, n, L, fill=0.0):
    out = torch.full((n, max(L, 1)) + tuple(v.shape[1:]), fill, dtype=v.dtype)
    return out.index_put((ray_id, pos), v)


def _rel_margin(q, thres):
    q = q.detach().double()
    return torch.where(q != 0, (q - thres).abs() / q.abs(), torch.full_like(q, math.inf))


# ---------------------------------------------------------------------------------------------------------------------
# samplers (fp32 points of the oracle's CPU ops)
# ---------------------------------------------------------------------------------------------------------------------
def _sample(P, ro, rd, kw, device='cpu'):
    kind, margins = P['kind'], {}
    if kind == 'dvgo':
        stepdist = float(kw['stepsize'] * P['voxel_size'])
        n_max = int((P['max_world_size'] - 1) / kw['stepsize']) + 1
        pts, outside, ray_id, step_id, *_ = CpuOps.sample_pts_on_rays(ro, rd, P['xyz_min'], P['xyz_max'], kw['near'], 1e9, stepdist)
        keep = ~outside
        return pts[keep], ray_id[keep], step_id[keep], n_max, {}, margins
    if kind == 'dmpigo':
        assert kw['near'] == 0 and kw['far'] == 1
        n_max = int((P['mpi_depth'] - 1) / kw['stepsize']) + 1
        pts, outside = CpuOps.sample_ndc_pts_on_rays(ro, rd, P['xyz_min'], P['xyz_max'], n_max)
        inside = ~outside
        n = inside.shape[0]
        ray_id = torch.arange(n).view(-1, 1).expand_as(inside)[inside]
        step_id = torch.arange(n_max).view(1, -1).expand_as(inside)[inside]
        return pts[inside], ray_id, step_id, n_max, {}, margins
    # DirectContractedVoxGO.sample_ray: the reference's fp32 torch expressions (lib/dcvgo.py:237-262), run on the device
    # the compared model runs on (the norm and the division round per device)
    ro, rd = ro.to(device), rd.to(device)
    o = (ro.float() - P['scene_center'].to(device)) / P['scene_radius'].to(device)
    d = rd.float() / rd.float().norm(dim=-1, keepdim=True)
    bg, wl, ss = P['bg_len'], P['world_len'], kw['stepsize']
    N_inner = int(2 / (2 + 2 * bg) * wl / ss) + 1
    b_inner = torch.linspace(0, 2, N_inner + 1, device=device)
    b_outer = 2 / torch.linspace(1, 1 / 128, N_inner + 1, device=device)
    t = torch.cat([(b_inner[1:] + b_inner[:-1]) * 0.5, (b_outer[1:] + b_outer[:-1]) * 0.5])
    pts = o[:, None, :] + d[:, None, :] * t[None, :, None]
    norm = pts.abs().amax(dim=-1, keepdim=True)
    inner = norm <= 1
    pts = torch.where(inner, pts, pts / norm * ((1 + bg) - bg / norm))
    pts, inner, t = pts.cpu(), inner.cpu(), t.cpu()
    keep = inner.squeeze(-1).clone()
    thres = (2 + 2 * bg) / wl * ss * 0.95
    dist = (pts[:, 1:] - pts[:, :-1]).norm(dim=-1).contiguous() if device == 'cpu' else \
        (pts[:, 1:].to(device) - pts[:, :-1].to(device)).norm(dim=-1).cpu().contiguous()
    keep[:, 1:] |= CpuOps.cumdist_thres(dist, thres)
    # the running sums the thresholded scan compares, in fp64 (reset after every emitted sample)
    cum = torch.zeros(dist.shape[0], dtype=torch.float64)
    m = torch.full(dist.shape[:1], math.inf, dtype=torch.float64)
    dd = dist.double()
    for i in range(dd.shape[1]):
        cum = cum + dd[:, i]
        m = torch.minimum(m, _rel_margin(cum, thres))
        cum = torch.where(cum > thres, torch.zeros_like(cum), cum)
    margins['cumdist'] = m
    n, n_max = keep.shape
    ray_id = torch.arange(n).view(-1, 1).expand(n, n_max)[keep]
    step_id = torch.arange(n_max).view(1, -1).expand(n, n_max)[keep]
    tt = t[None].expand(n, n_max)[keep]
    return pts[keep], ray_id, step_id, n_max, {'t': tt, 'inner': inner.squeeze(-1)[keep]}, margins


# ---------------------------------------------------------------------------------------------------------------------
# the forward
# ---------------------------------------------------------------------------------------------------------------------
def forward64(P, rays_o, rays_d, viewdirs, kw, global_step=None, is_train=False, rand_bkgd=None, sample_device='cpu'):
    """The reference's training forward in fp64.  rand_bkgd: callable(shape) -> the background draw (fp32 values) used
    when the model applies render_kwargs['rand_bkgd'].  sample_device: where DirectContractedVoxGO's sampler (torch
    arithmetic in the reference, not a kernel) runs.  Returns the reference's key set plus, under '_', the stages:
    per occupied sample its point / density, per composited sample alpha / T / liveness, per shaded sample its point /
    k0 / rgbnet input, and the threshold margins."""
    kind = P['kind']
    ro, rd, vd = (t.detach().cpu().float().contiguous() for t in (rays_o, rays_d, viewdirs))
    n = ro.shape[0]
    pts, ray_id, step_id, n_max, aux, margins = _sample(P, ro, rd, kw, sample_device)
    interval = float(kw['stepsize'] * P['voxel_size_ratio'])
    lo, hi = P['xyz_min'], P['xyz_max']

    occ = CpuOps.maskcache_lookup(P['mask'], pts.contiguous(), P['mask_scale'], P['mask_shift']) if pts.shape[0] else \
        torch.zeros(0, dtype=torch.bool)
    pts, ray_id, step_id = pts[occ], ray_id[occ], step_id[occ]
    aux = {k: v[occ] for k, v in aux.items()}

    density = grid_lookup(P['density'], pts, lo, hi)[:, 0]
    density.retain_grad()
    if kind == 'dmpigo':
        shift = grid_lookup(P['act_shift_grid'], pts, lo, hi)[:, 0].detach()
        x = density + shift
    else:
        shift = None
        x = density + P['act_shift']
    # 1 - (1 + e^x)^-interval; as 1 - exp(.) so that autograd's d alpha / dx = I sigma(x) (1 + e^x)^-I keeps its
    # digits when alpha rounds to 1 (expm1's backward, (result + 1) * grad, would cancel to 0)
    alpha = 1 - torch.exp(-interval * F.softplus(x))
    st = dict(occ_pts=pts, occ_ray_id=ray_id, occ_step_id=step_id, density=density, shift=shift, x=x.detach(),
              alpha_all=alpha.detach(), interval=interval)
    thres = P['fast_color_thres']
    raw_density = density
    if thres > 0:
        margins['alpha'] = _rel_margin(alpha, thres)
        sel = alpha.detach() > thres
        pts, ray_id, step_id, alpha, raw_density = pts[sel], ray_id[sel], step_id[sel], alpha[sel], raw_density[sel]
        aux = {k: v[sel] for k, v in aux.items()}
        st['sel_alpha'] = sel
    else:
        st['sel_alpha'] = torch.ones_like(ray_id, dtype=torch.bool)

    # transmittance: per ray, T_i = prod_{k<i} (1 - alpha_k); the scan stops after the first sample whose inclusive
    # product falls below 1e-3; later samples keep weight 0 and take no part in alphainv_last
    pos, L, counts = _segments(ray_id, n)
    A = _dense(alpha, ray_id, pos, n, L)
    Pin = torch.cumprod(1 - A, 1)
    Tex = torch.cat([torch.ones(n, 1, dtype=torch.float64), Pin[:, :-1]], 1)
    live_d = (Tex.detach() >= T_STOP)
    real = _dense(torch.ones_like(ray_id, dtype=torch.bool), ray_id, pos, n, L, False)
    live_d &= real
    T = Tex[ray_id, pos]
    live = live_d[ray_id, pos]
    weights = T * alpha * live
    alphainv_last = torch.where(live_d, 1 - A, torch.ones_like(A)).prod(1)
    margins['T'] = _rel_margin(Pin[ray_id, pos], T_STOP)[live]
    st.update(comp_ray_id=ray_id, comp_alpha=alpha.detach(), comp_T=T.detach(), comp_live=live, comp_pos=pos, counts=counts)
    if thres > 0:
        margins['weights'] = _rel_margin(weights, thres)
        sel = weights.detach() > thres
        pts, ray_id, step_id, alpha, weights, raw_density = (pts[sel], ray_id[sel], step_id[sel], alpha[sel], weights[sel],
                                                             raw_density[sel])
        aux = {k: v[sel] for k, v in aux.items()}
        st['sel_weights'] = sel
    else:
        st['sel_weights'] = torch.ones_like(ray_id, dtype=torch.bool)

    k0 = grid_lookup(P['k0'], pts, lo, hi)
    k0.retain_grad()
    feat = diffuse = None
    if P['rgbnet'] is None:
        logit = k0
    else:
        e = (vd.double().unsqueeze(-1) * P['viewfreq'].double()).flatten(-2)
        vemb = torch.cat([vd.double(), e.sin(), e.cos()], -1)[ray_id]
        if kind == 'dmpigo':
            p = ((pts.double() - lo.double()) / (hi.double() - lo.double())).flip((-1,)) * 2 - 1
            pe = (p.unsqueeze(-1) * P['posfreq'].double()).flatten(-2)
            feat = torch.cat([k0, p, pe.sin(), pe.cos(), vemb], -1)
        elif P['rgbnet_direct']:
            feat = torch.cat([k0, vemb], -1)
        else:
            feat = torch.cat([k0[:, 3:], vemb], -1)
            diffuse = k0[:, :3]
        h = feat
        for i, (w, b) in enumerate(P['rgbnet']):
            h = F.linear(h, w, b)
            if i + 1 < len(P['rgbnet']):
                h = act_fn(h, P['act'], P.get('gauss_a', A_GAUSS))
        logit = h if diffuse is None else h + diffuse
    rgb = torch.sigmoid(logit)
    st.update(pts=pts, ray_id=ray_id, k0=k0, feat=feat, logit=logit.detach(), diffuse=diffuse is not None)

    rgb_feature = torch.zeros(n, 3, dtype=torch.float64).index_add(0, ray_id, weights.unsqueeze(-1) * rgb)
    training = is_train if kind == 'dcvgo' else (global_step is not None)
    bg = None
    if kw.get('rand_bkgd', False) and training and kind != 'dvgo':
        bg = rand_bkgd(rgb_feature.shape).double()
        rgb_marched = rgb_feature + alphainv_last.unsqueeze(-1) * bg
    else:
        rgb_marched = rgb_feature + alphainv_last.unsqueeze(-1) * kw['bg']
    s = (step_id + 0.5) / n_max if kind != 'dcvgo' else 1 - 1 / (1 + aux['t'])
    ret = {'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched, 'rgb_feature': rgb_feature,
           'raw_alpha': alpha, 'raw_rgb': rgb, 'ray_id': ray_id}
    if kind != 'dvgo':
        ret.update(n_max=n_max, s=s)
    if kind == 'dcvgo':
        inner = aux['inner']
        ret.update(t=aux['t'], step_id=step_id, raw_density=raw_density,
                   wsum_mid=torch.zeros(n, dtype=torch.float64).index_add(0, ray_id[inner], weights[inner]))
    if kw.get('render_depth', False):
        ret['depth'] = torch.zeros(n, dtype=torch.float64).index_add(0, ray_id, (weights * s.double()).detach())
    st.update(step_id=step_id, s=s, bg=bg, bg_const=float(kw['bg']), margins=margins)
    if kind == 'dcvgo':
        st['inner'] = aux['inner']
    ret['_'] = st
    return ret


# ---------------------------------------------------------------------------------------------------------------------
# the composite loss of run_sr.py:523-546 (the same function on both sides)
# ---------------------------------------------------------------------------------------------------------------------
LOSS_WEIGHTS = dict(main=1.0, entropy_last=0.01, nearclip=1.0, distortion=0.01, rgbper=0.1)


def _segment_positions(ray_id):
    n = int(ray_id.max()) + 1
    counts = torch.bincount(ray_id, minlength=n)
    start = torch.cumsum(counts, 0) - counts
    return n, torch.arange(ray_id.numel(), device=ray_id.device) - start[ray_id], int(counts.max())


def flatten_eff_distloss(w, m, interval, ray_id):
    """torch_efficient_distloss.flatten_eff_distloss: per ray, sum_ij w_i w_j |m_i - m_j| + interval / 3 * sum_i w_i^2,
    summed and divided by ray_id.max() + 1; m sorted within a ray, so the pair term is 2 sum_i w_i (m_i W_<i - (wm)_<i).
    The exclusive prefix sums run per ray (a padded [rays, longest] layout), as the package's segment_cumsum does."""
    n, pos, L = _segment_positions(ray_id)
    m = m.to(w.dtype)
    W = torch.zeros(n, L, dtype=w.dtype, device=w.device).index_put((ray_id, pos), w)
    WM = torch.zeros(n, L, dtype=w.dtype, device=w.device).index_put((ray_id, pos), w * m)
    w_prefix = (torch.cumsum(W, 1) - W)[ray_id, pos]
    wm_prefix = (torch.cumsum(WM, 1) - WM)[ray_id, pos]
    loss_uni = (1 / 3) * interval * w.pow(2)
    loss_bi = 2 * w * (m * w_prefix - wm_prefix)
    return (loss_bi.sum() + loss_uni.sum()) / n


def composite_loss(out, target, n_rays, near_thres=None, weights=LOSS_WEIGHTS):
    """run_sr.py:523-546: MSE, entropy on alphainv_last, nearclip on raw_density (DirectContractedVoxGO), the
    distortion loss on weights / s / ray_id (models that return s), rgbper on raw_rgb with detached weights."""
    target = target.to(out['rgb_marched'].dtype)
    loss = weights['main'] * F.mse_loss(out['rgb_marched'], target)
    if weights['entropy_last'] > 0:
        pout = out['alphainv_last'].clamp(1e-6, 1 - 1e-6)
        loss = loss + weights['entropy_last'] * -(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean()
    if weights['nearclip'] > 0 and 't' in out and near_thres is not None:
        density = out['raw_density'][out['t'] < near_thres]
        if len(density):
            loss = loss + weights['nearclip'] * (density - density.detach()).sum()
    if weights['distortion'] > 0 and 's' in out and out['weights'].numel():
        loss = loss + weights['distortion'] * flatten_eff_distloss(out['weights'], out['s'], 1 / out['n_max'], out['ray_id'])
    if weights['rgbper'] > 0 and out['weights'].numel():
        rgbper = (out['raw_rgb'] - target[out['ray_id']]).pow(2).sum(-1)
        loss = loss + weights['rgbper'] * (rgbper * out['weights'].detach()).sum() / n_rays
    return loss


# ---------------------------------------------------------------------------------------------------------------------
# error bounds of the fp32 library against this restatement (the model is in test_gpu_train_grad.py's docstring)
# ---------------------------------------------------------------------------------------------------------------------
def _grid_err(grid, pts, lo, hi):
    """Bound on |fp32 trilinear - fp64 trilinear| at fp32 points, per channel [S, C]: 10u sum_k w_k |g_k| for the
    eight-term FMA chain and the corner weights' products, plus the voxel coordinate's rounding (ATen's
    ((p - min) / len * 2 - 1 + 1) / 2 * (size - 1): within 5u (size - 1) per axis, summed over the axes) times twice
    the largest |g| among the cell's corners (the interpolant's slope bound).  The nearest voxel's 3^3
    neighbourhood holds every corner of the cell, so that max comes from a max-pool and a nearest lookup."""
    g = grid.detach().abs()
    X, Y, Z = g.shape[2:]
    A = grid_lookup(g, pts, lo, hi)
    mx = F.max_pool3d(g, kernel_size=3, stride=1, padding=1)
    xyz = pts.double().reshape(1, 1, 1, -1, 3)
    ind = ((xyz - lo.double()) / (hi.double() - lo.double())).flip((-1,)) * 2 - 1
    M = F.grid_sample(mx, ind, mode='nearest', align_corners=True).reshape(g.shape[1], -1).T
    cterm = 5 * U * (X + Y + Z)
    return 10 * U * A + 2 * cterm * M, cterm


def _seg_suffix(v, ray_id, pos, n, L):
    """per sample, the sum of v over the later samples of its ray."""
    D = _dense(v.double(), ray_id, pos, n, L)
    incl = D.flip(1).cumsum(1).flip(1)
    return (incl - D)[ray_id, pos]


def _seg_prefix(v, ray_id, pos, n, L):
    D = _dense(v.double(), ray_id, pos, n, L)
    return (D.cumsum(1) - D)[ray_id, pos]


def _gauss_dact(z, a):
    return (z.abs() / (a * a)) * torch.exp(-z * z / (2 * a * a))


class Bounds:
    """Element-wise error bounds of every compared quantity, from the restatement's fp64 values after ``backward()``.
    Attributes (fp64, aligned with the restatement's lists): rel_alpha / rel_T / rel_w (the margins' yardsticks),
    alpha_occ [S0], weights / raw_alpha / raw_rgb [S2], alphainv_last / rgb_marched [N], g_density [S0], g_k0 [S2, C],
    params {name: flat bound}."""

    def __init__(self, P, out, target, n_rays, near_thres=None, lw=LOSS_WEIGHTS):
        st = out['_']
        kind, N, I = P['kind'], n_rays, st['interval']
        lo, hi = P['xyz_min'], P['xyz_max']
        tgt = target.detach().cpu().double()
        with torch.no_grad():
            # ---- density and alpha, every occupied sample [S0]
            pts0 = st['occ_pts']
            E_x, cterm_d = _grid_err(P['density'], pts0, lo, hi)
            E_x = E_x[:, 0]
            if kind == 'dmpigo':
                E_x = E_x + _grid_err(P['act_shift_grid'], pts0, lo, hi)[0][:, 0]
            x = st['x']
            E_x = E_x + U * x.abs()
            alpha = st['alpha_all']
            sig = torch.sigmoid(x)
            p = torch.exp(-I * F.softplus(x))                           # 1 - alpha, with its digits near alpha = 1
            dal = I * sig * p                                            # d alpha / d x
            d_alpha = dal * E_x + p * (I * (3 * sig + 1) * U + 8 * U) + U * alpha
            self.alpha_occ = d_alpha
            self.rel_alpha = torch.where(alpha > 0, d_alpha / alpha, torch.full_like(alpha, math.inf))

            # ---- transmittance, composited samples [S1]
            s1 = st['sel_alpha']
            rid1, pos1, live = st['comp_ray_id'], st['comp_pos'], st['comp_live']
            L1 = int(pos1.max()) + 1 if pos1.numel() else 1
            a1, T1, da1, p1 = st['comp_alpha'], st['comp_T'], d_alpha[s1], p[s1]
            rho = torch.where(live, da1 / p1.clamp_min(1e-300) + 2 * U, torch.zeros_like(a1))
            # the fp32 product of (1 - alpha_k) is within prod_k (1 + rho_k) of the fp64 one (log1p: a near-opaque
            # sample whose 1 - alpha rounds away entirely has rho >> 1, and exp(sum rho) would be meaningless)
            lrho = torch.log1p(rho)
            R_ex = _seg_prefix(lrho, rid1, pos1, N, L1)
            self.rel_T = torch.expm1(R_ex + lrho)[live]                  # the inclusive product the stop compares
            dT1 = T1 * torch.expm1(R_ex)
            w1 = T1 * a1 * live
            dw1 = (dT1 * a1 + (T1 + dT1) * da1 + U * w1) * live
            self.rel_w = torch.where(w1 > 0, dw1 / w1.clamp_min(1e-300), torch.zeros_like(w1))
            R_tot = torch.zeros(N, dtype=torch.float64).index_add_(0, rid1, lrho)
            n_r = torch.zeros(N, dtype=torch.float64).index_add_(0, rid1, live.double())
            # T_last as the product of the exact 1 - alpha (fp64 rounds alpha to 1 past 1 - 1e-16; its value then
            # reads 0 while its derivative, -T_i, does not)
            T_last = torch.exp(torch.zeros(N, dtype=torch.float64).index_add_(
                0, rid1, torch.where(live, torch.log(p1), torch.zeros_like(p1))))
            dT_last = T_last * torch.expm1(R_tot)
            self.alphainv_last = dT_last
            # the entropy loss clamps alphainv_last to [1e-6, 1 - 1e-6]: a third threshold, on the loss side
            self.clamp_margin = None
            if lw['entropy_last'] > 0:
                self.clamp_margin = torch.minimum(_rel_margin(T_last, 1e-6), _rel_margin(T_last, 1 - 1e-6))
                self.rel_T_last = torch.expm1(R_tot) + 2 * U

            # ---- shaded samples [S2]
            s2 = st['sel_weights']
            rid2 = st['ray_id']
            w2, dw2, a2, da2 = w1[s2], dw1[s2], a1[s2], da1[s2]
            self.weights, self.raw_alpha = dw2, da2
            pts2 = st['pts']
            E_k0, cterm_k = _grid_err(P['k0'], pts2, lo, hi)
            rgb = out['raw_rgb'].detach()
            layers = [(w.detach(), b.detach()) for w, b in (P['rgbnet'] or [])]
            acts = []
            if P['rgbnet'] is None:
                E_logit = E_k0
            else:
                feat = st['feat'].detach()
                cols = [E_k0[:, 3:] if st['diffuse'] else E_k0]
                if kind == 'dmpigo':
                    fr = P['posfreq'].double()
                    cols += [torch.full((feat.shape[0], 3), 4 * U, dtype=torch.float64),
                             (4 * U * (1 + 2 * fr)).repeat(3).expand(feat.shape[0], -1).repeat(1, 2)]
                vf = P['viewfreq'].double()
                cols += [torch.full((feat.shape[0], 3), 2 * U, dtype=torch.float64),
                         (4 * U * (1 + 2 * vf)).repeat(3).expand(feat.shape[0], -1).repeat(1, 2)]
                E = torch.cat(cols, 1)
                assert E.shape == feat.shape
                h = feat
                a_g = float(np.float32(P.get('gauss_a', A_GAUSS)))
                for i, (W, b) in enumerate(layers):
                    z = h @ W.T + b
                    S = (h.abs() + E) @ W.abs().T + b.abs()
                    Ez = E @ W.abs().T + (W.shape[1] + 2) * U * S
                    acts.append((h, E))
                    if i + 1 < len(layers):
                        if P['act'] == 'gauss':
                            g, Eg = mpi_act_step(z.numpy(), Ez.numpy(), a_g)
                            g, Eg = torch.from_numpy(g), torch.from_numpy(Eg)
                        else:
                            g = act_fn(z, P['act'])
                            Eg = Ez + U * g.abs()
                        acts[-1] = acts[-1] + (z, Ez)
                        h, E = g, Eg
                    else:
                        acts[-1] = acts[-1] + (z, Ez)
                E_logit = Ez
                if st['diffuse']:
                    E_logit = E_logit + E_k0[:, :3] + U * st['logit'].abs()
            E_rgb = 0.25 * E_logit + 2 * U * rgb
            self.raw_rgb = E_rgb
            nr2 = n_r[rid2]
            feat_r = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, rid2, dw2[:, None] * rgb + w2[:, None] * E_rgb)
            mag_feat = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, rid2, w2[:, None] * rgb)
            bg = st['bg'] if st['bg'] is not None else torch.full((N, 3), st['bg_const'], dtype=torch.float64)
            E_rgbm = feat_r + (n_r[:, None] + 1) * U * mag_feat + dT_last[:, None] * bg.abs() + \
                2 * U * (mag_feat + T_last[:, None] * bg.abs())
            self.rgb_marched = E_rgbm

            # ---- the loss's upstream gradients
            rgbm = out['rgb_marched'].detach()
            c_m = 2 * lw['main'] / (3 * N)
            g_rgbm = c_m * (rgbm - tgt)
            E_grgbm = c_m * (E_rgbm + 2 * U * (rgbm.abs() + tgt.abs()))
            g_last = (g_rgbm * bg).sum(1)
            E_glast = (E_grgbm * bg.abs()).sum(1) + 4 * U * (g_rgbm * bg).abs().sum(1)
            if lw['entropy_last'] > 0:
                pl = T_last
                act_e = (pl > 1e-6) & (pl < 1 - 1e-6)
                lp, l1p = torch.log(pl.clamp(1e-6, 1 - 1e-6)), torch.log1p(-pl.clamp(1e-6, 1 - 1e-6))
                ce = lw['entropy_last'] / N
                g_e = torch.where(act_e, ce * (l1p - lp), torch.zeros_like(pl))
                E_e = torch.where(act_e, ce * (dT_last / (pl * (1 - pl)).clamp_min(1e-300) +
                                               4 * U * (lp.abs() + l1p.abs() + 1)), torch.zeros_like(pl))
                g_last, E_glast = g_last + g_e, E_glast + E_e + 4 * U * g_e.abs()
            D = torch.zeros_like(w2)
            E_D = torch.zeros_like(w2)
            if lw['distortion'] > 0 and kind != 'dvgo' and w2.numel():
                s = st['s'].double()
                pos2, L2, _ = _segments(rid2, N)
                Wd, Sd, dWd = (_dense(v, rid2, pos2, N, L2) for v in (w2, s, dw2))
                absd = (Sd[:, :, None] - Sd[:, None, :]).abs()
                real2 = _dense(torch.ones_like(rid2, dtype=torch.bool), rid2, pos2, N, L2, False)
                absd = absd * real2[:, :, None] * real2[:, None, :]
                pair = (absd * Wd[:, None, :]).sum(2)[rid2, pos2]
                dpair = (absd * dWd[:, None, :]).sum(2)[rid2, pos2]
                cd = lw['distortion'] / (int(rid2.max()) + 1)
                Id = 1.0 / out['n_max']
                D = cd * (2 * pair + (2 / 3) * Id * w2)
                E_D = cd * (2 * dpair + (2 / 3) * Id * dw2) + (4 * nr2 + 8) * U * D
            g_w = (g_rgbm[rid2] * rgb).sum(1) + D
            E_gw = (E_grgbm[rid2] * rgb + g_rgbm[rid2].abs() * E_rgb).sum(1) + E_D + \
                4 * U * ((g_rgbm[rid2].abs() * rgb).sum(1) + D)
            crp = 2 * lw['rgbper'] / N
            g_rgb = w2[:, None] * g_rgbm[rid2] + crp * (rgb - tgt[rid2]) * w2[:, None]
            E_grgb = dw2[:, None] * g_rgbm[rid2].abs() + w2[:, None] * E_grgbm[rid2] + \
                crp * (dw2[:, None] * (rgb - tgt[rid2]).abs() + w2[:, None] * E_rgb) + \
                4 * U * (w2[:, None] * g_rgbm[rid2].abs() + crp * w2[:, None] * (rgb.abs() + tgt[rid2].abs()))

            # ---- Alphas2Weights.backward on the composited list [S1]
            g_w1 = torch.zeros_like(a1).masked_scatter_(s2, g_w)
            E_gw1 = torch.zeros_like(a1).masked_scatter_(s2, E_gw)
            gwl = g_w1 * w1
            B = _seg_suffix(gwl, rid1, pos1, N, L1) + g_last[rid1] * T_last[rid1]
            magB = _seg_suffix(g_w1.abs() * w1, rid1, pos1, N, L1) + g_last[rid1].abs() * T_last[rid1]
            E_B = _seg_suffix(E_gw1 * w1 + g_w1.abs() * dw1, rid1, pos1, N, L1) + E_glast[rid1] * T_last[rid1] + \
                g_last[rid1].abs() * dT_last[rid1] + (n_r[rid1] + 2) * U * magB
            # B / (1 - alpha): 1 - alpha's relative error da / (1 - alpha) and the kernel's + 1e-10; when fp32 cannot
            # resolve 1 - alpha at all (alpha rounds to 1, later weights and T_last to 0) the kernel's term is 0, an
            # error of the whole term at most
            om = p1.clamp_min(1e-300)
            g_a = (g_w1 * T1 - B / om) * live
            # (B and every later term carry the factor 1 - alpha: |B| / (1 - alpha) <= magB / (1 - alpha) stays
            # finite, and the kernel's quotient lies between 0 and that, times the prior T's error)
            cond = (da1 + 1e-10) / om
            term = torch.where(cond < 1, E_B / om + magB / om * cond, 2 * magB / om * (1 + torch.expm1(R_ex)))
            E_ga = (E_gw1 * T1 + g_w1.abs() * dT1 + term + 3 * U * (g_w1.abs() * T1 + magB / om)) * live
            # ---- Raw2Alpha.backward [S0]
            g_a0 = torch.zeros_like(alpha).masked_scatter_(s1, g_a)
            E_ga0 = torch.zeros_like(alpha).masked_scatter_(s1, E_ga)
            d_dal = U * ((I + 1) * (3 + x.abs()) + 10) + (1 + I) * E_x
            # fp32 underflow: (1 + e^x)^(-I-1) below the normal range (2^-126) and a result below 2^-149
            self.g_density = E_ga0 * dal + g_a0.abs() * (dal * d_dal + I * (torch.exp(x) + 1) * 2.0 ** -126) + 2.0 ** -149
            near0 = torch.zeros_like(alpha)
            if lw['nearclip'] > 0 and kind == 'dcvgo' and near_thres is not None and w2.numel():
                # nearclip's constant joins the sample's gradient in one fp32 addition
                near2 = (out['t'] < near_thres).double() * lw['nearclip']
                near1 = torch.zeros_like(a1).masked_scatter_(s2, near2)
                near0 = torch.zeros_like(alpha).masked_scatter_(s1, near1)
                self.g_density = self.g_density + U * ((g_a0 * dal).abs() + self.g_density + near0) * (near0 > 0)

            # ---- colour branch backward [S2]
            sp = rgb * (1 - rgb)
            g_logit = g_rgb * sp
            E_glogit = E_grgb * sp + g_rgb.abs() * (0.1 * E_logit + 3 * U * sp)
            self.params = {}
            S2 = w2.shape[0]
            if P['rgbnet'] is None:
                g_k0, E_gk0 = g_logit, E_glogit
            else:
                dl, Edl = g_logit, E_glogit
                for i in range(len(layers) - 1, -1, -1):
                    W, b = layers[i]
                    h, Eh = acts[i][0], acts[i][1]
                    self.params[f'rgbnet.L{i}.weight'] = (Edl.T @ h.abs() + dl.abs().T @ Eh +
                                                          (S2 + 2) * U * dl.abs().T @ h.abs()).flatten()
                    self.params[f'rgbnet.L{i}.bias'] = Edl.sum(0) + (S2 + 2) * U * dl.abs().sum(0)
                    dh = dl @ W
                    Edh = Edl @ W.abs() + (W.shape[0] + 2) * U * dl.abs() @ W.abs()
                    if i > 0:
                        z, Ez = acts[i - 1][2], acts[i - 1][3]
                        if P['act'] == 'gauss':
                            gp = -z / (a_g * a_g) * torch.exp(-z * z / (2 * a_g * a_g))
                            ddg = Ez / (a_g * a_g) + 4 * U * gp.abs()
                        else:
                            slope = 0.0 if P['act'] == 'relu' else float(np.float32(0.01))
                            gp = torch.where(z > 0, torch.ones_like(z), torch.full_like(z, slope))
                            ddg = torch.where(z.abs() <= Ez, torch.full_like(z, 1 - slope), torch.zeros_like(z))
                        dl = dh * gp
                        Edl = Edh * gp.abs() + dh.abs() * ddg + U * dl.abs()
                nk = P['k0'].shape[1] - (3 if st['diffuse'] else 0)
                g_k0, E_gk0 = dh[:, :nk], Edh[:, :nk]
                if st['diffuse']:
                    g_k0, E_gk0 = torch.cat([g_logit, g_k0], 1), torch.cat([E_glogit, E_gk0], 1)
            self.g_k0 = E_gk0

            # ---- scatter into the grids
            def grid_bound(grid, pts_, g_s, E_s, cterm):
                C, X, Y, Z = grid.shape[1:]
                idx, wc = corners(pts_, lo, hi, (X, Y, Z))
                nvox = X * Y * Z
                out_ = torch.zeros(C, nvox, dtype=torch.float64)
                cnt = scatter_corners((wc > 0).double(), idx, nvox)
                for c in range(C):
                    ag = g_s[:, c].abs()[:, None]
                    main = scatter_corners(wc * E_s[:, c][:, None], idx, nvox)
                    coord = scatter_corners((2 * cterm + 4 * U) * ag.expand(-1, 8) * (wc >= 0), idx, nvox)
                    summ = scatter_corners(wc * ag, idx, nvox)
                    out_[c] = main + coord + (cnt + 2) * U * summ
                return out_.flatten(), cnt

            g_d_all = g_a0 * dal + near0
            self.params['density.grid'], self.count_density = grid_bound(P['density'], pts0, g_d_all[:, None],
                                                                         self.g_density[:, None], cterm_d)
            self.params['k0.grid'], self.count_k0 = grid_bound(P['k0'], pts2, g_k0, E_gk0, cterm_k)
            self.n_r, self.R_tot = n_r, R_tot


def mpi_act_step(z, E, a):
    """mpi_act._act_step for the Gaussian in fp32 (tests/mpi_act.py: the mean value theorem on [z - E, z + E] plus the
    fp32 evaluation of exp(-z^2 / 2a^2))."""
    import mpi_act
    return mpi_act._act_step(z, E, 'gauss', a, False)


def check_margins(P, b, out):
    """Every threshold decision must be farther from its threshold than the fp32 error of the compared quantity:
    returns the list of violations (empty: fp32 and fp64 take every sample to the same fate)."""
    st = out['_']
    m = st['margins']
    bad = []
    if 'alpha' in m:
        v = m['alpha'] <= b.rel_alpha
        if v.any():
            bad.append(('alpha > fast_color_thres', int(v.sum()), float(m['alpha'][v].min())))
    v = m['T'] <= b.rel_T
    if v.any():
        bad.append(('T < 1e-3', int(v.sum()), float(m['T'][v].min())))
    if 'weights' in m:
        v = m['weights'] <= b.rel_w
        if v.any():
            bad.append(('weights > fast_color_thres', int(v.sum()), float(m['weights'][v].min())))
    if b.clamp_margin is not None:
        v = b.clamp_margin <= b.rel_T_last
        if v.any():
            bad.append(('alphainv_last at the entropy clamp', int(v.sum()), float(b.clamp_margin[v].min())))
    if 'cumdist' in m:
        v = m['cumdist'] <= 8 * U
        if v.any():
            bad.append(('cumdist > thres', int(v.sum()), float(m['cumdist'][v].min())))
    return bad
