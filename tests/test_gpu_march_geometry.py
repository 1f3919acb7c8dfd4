"""GPU: the marchers' ray geometry, occupancy lookup, empty-space skipping and compositing, per ray, on scenes that are
not centred, not cubic and not isotropic, with an occupancy mask of its own resolution and with edge rays.

Every case renders with the CPU oracle (oracle.pipeline.forward on ops.CpuOps; also on RefExtOps, the reference's own
kernels, where oracle/_ref was built) and with every marcher mode its shape has, in 2-D tile order and in linear order,
and with empty-space skipping on and off.  Checks per ray:

  * geometry, bit for bit: the step count and t_min / t_max (DirectVoxGO), and the numbers of in-box samples S_m,
    occupancy hits S_d and -- with a threshold -- shaded samples S_c.  The one exception is a ray on which a
    value-dependent decision is borderline: T within rounding of the 1e-3 early-out, or an alpha / weight within rounding
    of fast_color_thres (expf / powf differ by a few ulp between the CUDA math library and the host libm).  Such a ray
    is named and must be shown to be borderline (BORDER) from the oracle's trace; at most floor(1e-4 N) of them per
    render, so none at the sizes used here.
    Skipping on and off must give identical outputs and ray_stats.
  * values, fp32 mode against a float64 recomposition of the same ray from the oracle's trace (fp64_reference): rgb,
    depth and alphainv_last within a bound built from that ray's own samples.
  * tensor-core modes against fp32 mode with the bound of test_gpu_march_mlp.check_per_ray_against_fp32.

Error model of the recomposition (u = 2^-24):
  * density: the marcher's trilinear sum (k4_march_common.cuh) and the oracle's CPU grid_sample use the same fp32 corner
    weights and round the eight-term sum differently (FMA chain against separate products and adds); each is within
    8 u S of the exact sum, S = sum_k |v_k| w_k, so they differ by at most DEN_REL * u * S with DEN_REL = 16.  (An fp32
    emulation of the marcher's arithmetic on the CPU differed from grid_sample by at most 3.4 u S on 20,000 points.)
  * alpha = 1 - powf(1 + expf(d + shift), -interval): the add u; expf and powf within EXPF_ULP = 2 and POWF_ULP = 4 ulp
    (CUDA C++ Programming Guide, single-precision mathematical functions, maximum ulp error, full range); 1 + e u; the
    final subtraction u.  Carried through an interval [alpha_lo, alpha_hi] per sample.
  * T and w: every T update rounds once (the product is taken in double), w = T * alpha once; the interval bounds are
    carried along the ray.
  * colour: the fp32 rgbnet bound (march_bounds.true_logit_bound), the sigmoid (SIG_REL), the product w * sigma, the
    sequential sum of n terms ((n - 1) u sum), the background product T * bg and the final add.
"""
import ctypes as C
import itertools
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ops, pipeline, scenes
from helpers import model_from_state
from march_bounds import FEAT_REL, SIG_REL, U, sig, true_logit_bound, types_ns

pytestmark = pytest.mark.gpu

DEN_REL = 16.0        # GPU against oracle density, in u * S (module docstring)
EXPF_ULP = 2.0
POWF_ULP = 4.0
ULP = 2.0 ** -23      # one ulp relative to the value, at most
BORDER = 16 * ULP     # "within rounding" of a threshold: expf / powf ulp errors carried through a few roundings
RATIOS = {}           # largest error / bound per check and scene, printed as the cases run


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
BOX_A = ([-0.7, -1.3, -0.2], [1.1, 0.4, 0.9])                 # off-centre, non-cubic
BOX_B = ([-0.75, -1.25, -0.5], [1.25, 0.5, 0.875])            # off-centre, with dyadic extents: exact mask scale / shift
FG_BOX = ([-0.6, -1.2, -0.3], [1.0, 0.5, 0.9])                # DCVGO foreground: centre (0.2, -0.35, 0.3), radii .8 .85 .6
MPI_BOX = ([-1.3, -1.9, -1.0], [1.7, 1.2, 0.9])
RGBNET = dict(rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4)     # wgmma configuration 1 (exact shape)
MPI_RGBNET = dict(rgbnet_dim=9, rgbnet_depth=3, rgbnet_width=64, viewbase_pe=0, spatial_pe=0)   # wgmma configuration 6


def _num_voxels(box, dims):
    """num_voxels for which DirectVoxGO's world size comes out as dims (lib/dvgo.py:152-158)."""
    ln = np.subtract(box[1], box[0])
    vs = np.mean([ln[a] / (dims[a] + 0.5) for a in range(3)])
    return int(round(float(np.prod(ln)) / vs ** 3))


SPARSE = 0.99985      # seed density of the masks with their own resolution: empty regions several skip cells wide


def _blobs(ws, seed, p=0.9985):
    g = torch.Generator().manual_seed(seed)
    seeds = (torch.rand(ws, generator=g) > p).float()[None, None]
    return F.max_pool3d(seeds, kernel_size=5, stride=1, padding=2)[0, 0] > 0


def _voxel_of(st, xyz):
    ws = st['density'].shape[2:]
    mn, mx = st['xyz_min'].tolist(), st['xyz_max'].tolist()
    return [min(max(int(round((xyz[a] - mn[a]) / (mx[a] - mn[a]) * (ws[a] - 1))), 1), ws[a] - 2) for a in range(3)]


def _patches(st, sat_at, dead_at):
    """A 3^3-voxel patch of saturating density (den + shift > 89: expf overflows, alpha = 1 exactly) and one of dead
    density (expf underflows, alpha = 0 exactly), both occupied."""
    den = st['density'][0, 0]
    for xyz, v in ((sat_at, 120.0), (dead_at, -200.0)):
        i, j, k = _voxel_of(st, xyz)
        den[i - 1:i + 2, j - 1:j + 2, k - 1:k + 2] = v
        if tuple(st['mask_cache']['mask'].shape) == tuple(den.shape):
            st['mask_cache']['mask'][i - 1:i + 2, j - 1:j + 2, k - 1:k + 2] = True


def dvgo_scene(box, dims, regime, thres, mask_dims=None, seed=0):
    st = pipeline.dvgo_state(*box, num_voxels=_num_voxels(box, dims), num_voxels_base=_num_voxels(box, dims),
                             alpha_init=1e-2, fast_color_thres=thres, rgbnet_direct=True, **RGBNET)
    assert st['density'].shape[2:] == tuple(dims), (st['density'].shape, dims)
    st.update(_num_voxels=_num_voxels(box, dims), _num_voxels_base=_num_voxels(box, dims), _alpha_init=1e-2)
    scenes.fill_grids(st, 'fog' if regime == 'blobs' else regime)
    scenes.fill_rgbnet(st)
    if regime == 'blobs':
        b = _blobs(list(dims), seed)
        st['density'] = torch.where(b, torch.full(dims, 3.0), torch.full(dims, -6.0))[None, None].contiguous()
        st['mask_cache'] = pipeline.mask_grid_state(b, st['xyz_min'], st['xyz_max'])
    if mask_dims is not None:
        st['mask_cache'] = pipeline.mask_grid_state(_blobs(list(mask_dims), seed + 7, p=SPARSE), st['xyz_min'], st['xyz_max'])
    _patches(st, (0.05, -0.1, 0.15), (0.6, -0.8, 0.6))
    st['fast_color_thres'] = thres
    return st


def mpi_scene(regime, mask_dims=None, seed=0):
    xy, depth = 40, 24
    st = pipeline.dmpigo_state(*MPI_BOX, num_voxels=xy * xy * depth, mpi_depth=depth, fast_color_thres=1.0 / depth / 5,
                               **MPI_RGBNET)
    st['_num_voxels'] = xy * xy * depth
    scenes.fill_grids(st, regime)
    scenes.fill_rgbnet(st)
    if mask_dims is not None:
        st['mask_cache'] = pipeline.mask_grid_state(_blobs(list(mask_dims), seed + 3, p=SPARSE), st['xyz_min'], st['xyz_max'])
    return st


def dcvgo_scene(regime):
    res, bg_len = 40, 0.2
    st = pipeline.dcvgo_state(*FG_BOX, num_voxels=res ** 3, num_voxels_base=res ** 3, alpha_init=1e-2,
                              fast_color_thres=1e-4, bg_len=bg_len, rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=128,
                              viewbase_pe=4)
    st['kind'] = 'dvgo'
    scenes.fill_grids(st, regime)
    st['kind'] = 'dcvgo'
    scenes.fill_rgbnet(st)
    st.update(_num_voxels=res ** 3, _num_voxels_base=res ** 3, _alpha_init=1e-2, _fg_min=FG_BOX[0], _fg_max=FG_BOX[1])
    return st


# ---------------------------------------------------------------------------------------------------------------------
# rays
# ---------------------------------------------------------------------------------------------------------------------
def orbit(H, W, **kw):
    ro, rd, vd = scenes.blender_rays(H, W, **kw)
    return ro, rd, vd, (H, W)


def _rays(o, d):
    o = torch.tensor(o, dtype=torch.float32)
    d = torch.tensor(d, dtype=torch.float32)
    return o, d, d / d.norm(dim=-1, keepdim=True)


def tie_coord(st, a, k):
    """A world coordinate on axis a that maps exactly to k + 1/2 in the mask's voxel coordinates (k even: roundf gives
    k + 1, rintf k), or None when the mask's scale and shift do not allow one."""
    sc = float(st['mask_cache']['xyz2ijk_scale'][a])
    sh = float(st['mask_cache']['xyz2ijk_shift'][a])
    c = np.float32((k + 0.5 - sh) / sc)
    return float(c) if float(c) * sc + sh == k + 0.5 else None


def edge_rays(st):
    """Rays of DirectVoxGO geometry's edges, with the indices of the special ones:
      tie   axis-parallel rays (two zero direction components) whose constant coordinates lie exactly on mask half-voxels
      face  a -x ray whose first sample lies exactly on xyz_max[0], with y on the xyz_min[1] face
      one   a ray with one zero component
      far   a ray that misses the box with an entry parameter beyond 1e9 (t_min / t_max clamp at `far` = 1e9)"""
    mn, mx = st['xyz_min'].tolist(), st['xyz_max'].tolist()
    mdims = st['mask_cache']['mask'].shape
    ks = [2 * (m // 4) for m in mdims]                  # even, inside the mask
    ties = [tie_coord(st, a, ks[a]) for a in range(3)]
    mid = [0.5 * (mn[a] + mx[a]) for a in range(3)]
    t = [ties[a] if ties[a] is not None else mid[a] + 0.013 for a in range(3)]
    o, d, idx = [], [], {}
    idx['tie'] = list(range(0, 3))
    o += [[mn[0] - 0.5, t[1], t[2]], [t[0], mx[1] + 0.5, t[2]], [t[0], t[1], mn[2] - 0.5]]
    d += [[1, 0, 0], [0, -1, 0], [0, 0, 2]]
    idx['face'] = [3]
    o += [[2 * mx[0], mn[1], t[2]]]                     # t_min = xyz_max[0] exactly, so the first sample is on that face
    d += [[-1, 0, 0]]
    idx['one'] = [4, 5]
    o += [[mn[0] - 0.3, t[1], mn[2] - 0.4], [mid[0], mn[1] - 0.3, mid[2] + 0.1]]
    d += [[0.6, 0, 0.8], [0.2, 0.9, 0]]
    idx['far'] = [6]
    o += [[mid[0], mx[1] + 4.0, mid[2]]]
    d += [[1.0, -1e-9, 0.3]]
    ro, rd, vd = _rays(o, d)
    return ro, rd, vd, (1, ro.shape[0]), idx, ties


# ---------------------------------------------------------------------------------------------------------------------
# running
# ---------------------------------------------------------------------------------------------------------------------
def ref_ext_ops(kind, monkeypatch):
    """The reference's own kernels where oracle/_ref was built (else None), with TF32 off for this test only."""
    if not os.path.exists(ops.ref_ext_path()):
        return None
    if kind == 'dcvgo' and not os.path.exists(os.path.join(os.path.dirname(ops.ref_ext_path()), 'ub360_utils_cuda.so')):
        return None
    monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    return ops.RefExtOps()


def models(st, dev, monkeypatch):
    """{True: model with empty-space skipping, False: without} (DirectContractedVoxGO has no skipping)."""
    out = {}
    for skip in ((True, False) if st['kind'] != 'dcvgo' else (True,)):
        if skip:
            monkeypatch.delenv('K4_NO_SKIP', raising=False)
        else:
            monkeypatch.setenv('K4_NO_SKIP', '1')          # read by k4_scene_create
        m = model_from_state(st, dev)
        m._get_scene()
        out[skip] = m
    monkeypatch.delenv('K4_NO_SKIP', raising=False)
    return out


def modes_of(st):
    if st['kind'] == 'dcvgo':
        return ('fp32', 'f16', 'f16x3', 'ws', 'auto')
    if st['rgbnet'] is None:
        return ('fp32', 'auto')
    return ('fp32', 'f16', 'f16x3', 'ws')


def render_all(ms, ro, rd, vd, kw, hw, modes):
    dev = ms[True].density.grid.device
    ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
    outs = {}
    for skip, m in ms.items():
        for mode in modes:
            for order in (hw, None):
                o = m.render_rays(ro, rd, vd, kw, image_hw=order, mlp_mode=mode, debug=True)
                outs[(skip, mode, order)] = o
    torch.cuda.synchronize()
    return {k: {n: t.cpu() for n, t in o.items()} for k, o in outs.items()}


def borderline(r, trace, thres):
    """True when a value-dependent decision of ray r is within rounding in the oracle's trace."""
    c, oc = trace['composited'], trace['occupied']
    sel = c['ray_id'] == r
    T, a = c['T'][sel].double(), c['alpha'][sel].double()
    after = T * (1 - a)
    if bool(((after / 1e-3 - 1).abs() <= BORDER).any()):
        return True
    if thres > 0:
        ao = oc['alpha'][oc['ray_id'] == r].double()
        if bool(((ao / thres - 1).abs() <= BORDER).any()) or bool((((T * a) / thres - 1).abs() <= BORDER).any()):
            return True
    return False


def check_geometry(out, ref, trace, st, N, label):
    """Per-ray geometry against the oracle (module docstring); returns the borderline rays, which the value checks skip."""
    rs = out['ray_stats'].long()
    ors = ref['_ray_stats'].cpu().long()
    thres = float(st['fast_color_thres'])
    n_c = torch.bincount(trace['ray_id'].cpu().long(), minlength=N)
    diff = (rs[:, 1] != ors[:, 0]) | (rs[:, 2] != ors[:, 1])
    if thres > 0:
        diff |= rs[:, 3] != n_c                        # without a threshold the oracle shades past the early-out
    if st['kind'] == 'dvgo':
        assert torch.equal(rs[:, 0], ref['_N_steps'].cpu().long()), (label, 'step counts')
        tm = out['t_minmax']
        assert torch.equal(tm[:, 0], ref['_t_min'].cpu()) and torch.equal(tm[:, 1], ref['_t_max'].cpu()), (label, 't_min/t_max')
    bad = diff.nonzero().flatten().tolist()
    assert len(bad) <= int(1e-4 * N), (label, 'rays with different sample counts', bad[:20])
    for r in bad:
        assert borderline(r, trace, thres), (label, 'ray', r, 'ours', rs[r].tolist(), 'oracle', ors[r].tolist(), int(n_c[r]))
    return bad


# ---------------------------------------------------------------------------------------------------------------------
# float64 recomposition of every ray from the oracle's trace
# ---------------------------------------------------------------------------------------------------------------------
def _abs_interp(st, key, pts):
    if pts.shape[0] == 0:
        return torch.zeros(0, dtype=torch.float64)
    g = st[key].double().abs()
    return pipeline.dense_grid(g, pts.double(), st['xyz_min'].double(), st['xyz_max'].double()).reshape(pts.shape[0], -1).sum(-1)


def _alpha(x, interval):
    """1 - (1 + e^x)^-interval in float64, accurate for alpha near 0 and near 1."""
    with np.errstate(over='ignore'):
        lp = np.where(x > 30, x + np.log1p(np.exp(-np.minimum(x, 700))), np.log1p(np.exp(np.minimum(x, 30))))
    return -np.expm1(-interval * lp)


def _alpha_bounds(x64, dx, interval):
    """[alpha_lo, alpha_hi] of the marcher's fp32 alpha for a pre-activation within dx of x64 (module docstring)."""
    lo, hi = x64 - dx, x64 + dx
    with np.errstate(over='ignore'):
        e_lo = np.exp(np.minimum(lo, 700)) * (1 - EXPF_ULP * ULP)
        e_hi = np.exp(np.minimum(hi, 700)) * (1 + EXPF_ULP * ULP)
    e_hi = np.where(e_hi * (1 - ULP) >= 2.0 ** 128 * (1 - 2.0 ** -25), np.inf, e_hi)     # expf overflows: inf, alpha = 1
    b_lo, b_hi = (1 + e_lo) * (1 - U), (1 + e_hi) * (1 + U)
    with np.errstate(divide='ignore'):
        p_hi = np.exp(-interval * np.log(b_lo)) * (1 + POWF_ULP * ULP)
        p_lo = np.where(np.isinf(b_hi), 0.0, np.exp(-interval * np.log(b_hi)) * (1 - POWF_ULP * ULP))
    a_lo = np.clip((1 - p_hi) * (1 - U), 0, 1)
    a_hi = np.clip((1 - p_lo) * (1 + U), 0, 1)
    return a_lo, a_hi


def interval_of(st, kw):
    if st['kind'] == 'dmpigo':
        return float(np.float32(kw['stepsize'] * st['voxel_size_ratio']))
    return float(np.float32(np.float32(kw['stepsize']) * np.float32(float(st['voxel_size_ratio']))))


def fp64_reference(st, trace, N, kw, skip_rays):
    """Per ray: rgb, depth and alphainv_last recomposed in float64 from the oracle's trace, and their bounds against
    fp32 mode.  Rays in skip_rays (borderline decisions) get an infinite bound."""
    oc, cp = trace['occupied'], trace['composited']
    shift = 0.0 if st['kind'] == 'dmpigo' else float(st['act_shift'])
    I = interval_of(st, kw)
    # per occupied sample: x = density + shift, and how far the marcher's may lie from it
    S = _abs_interp(st, 'density', oc['pts'])
    if st['kind'] == 'dmpigo':
        S = S + _abs_interp(st, 'act_shift_grid', oc['pts'])
    d = oc['density'].double().numpy()
    x64 = d + shift
    dx = DEN_REL * U * S.numpy() + U * (np.abs(x64) + 2 * np.abs(d))
    a_lo, a_hi = _alpha_bounds(x64, dx, I)
    a64 = _alpha(x64, I)
    big = 1 << 32
    okey = (oc['ray_id'].long() * big + oc['step_id'].long()).numpy()
    ckey = (cp['ray_id'].long() * big + cp['step_id'].long()).numpy()
    ci = np.searchsorted(okey, ckey)
    assert np.array_equal(okey[ci], ckey)
    # composite every ray up to the oracle's early-out, carrying [T_lo, T_hi] and [w_lo, w_hi]
    crid = cp['ray_id'].long().numpy()
    nC = ckey.shape[0]
    w64, w_lo, w_hi = np.zeros(nC), np.zeros(nC), np.zeros(nC)
    T64, T_lo, T_hi = np.ones(N), np.ones(N), np.ones(N)
    i_end = cp['i_end'].long().numpy()
    starts = np.searchsorted(crid, np.arange(N))
    for r in np.unique(crid):
        s, e = int(starts[r]), int(i_end[r])
        if e <= s:
            continue
        A64, Alo, Ahi = a64[ci[s:e]], a_lo[ci[s:e]], a_hi[ci[s:e]]
        f64 = np.cumprod(np.concatenate([[1.0], 1 - A64]))
        flo = np.cumprod(np.concatenate([[1.0], (1 - Ahi) * (1 - U)]))
        fhi = np.cumprod(np.concatenate([[1.0], np.minimum((1 - Alo) * (1 + U), 1.0)]))
        w64[s:e] = f64[:-1] * A64
        w_lo[s:e] = flo[:-1] * Alo * (1 - U)
        w_hi[s:e] = fhi[:-1] * Ahi * (1 + U)
        T64[r], T_lo[r], T_hi[r] = f64[-1], flo[-1], fhi[-1]
    dT = np.maximum(T_hi - T64, T64 - T_lo) * (1 + 1e-9)
    # shaded samples
    skey = (trace['ray_id'].long() * big + trace['step_id'].long()).numpy()
    si = np.searchsorted(ckey, skey)
    assert np.array_equal(ckey[si], skey)
    srid = trace['ray_id'].long().numpy()
    ws64, wslo, wshi = w64[si], w_lo[si], w_hi[si]
    dw = np.maximum(wshi - ws64, ws64 - wslo)[:, None]
    x = trace['rgb_feat'].double().numpy()
    D0 = FEAT_REL * np.abs(x) + 2.0 ** -24
    if st['rgbnet'] is None:
        lg, E = x, D0
    else:
        shp = types_ns(st)
        diff = None if trace['diffuse'] is None else trace['diffuse'].double().numpy()
        lg, E = true_logit_bound('fp32', shp, x, diff, D0)
    zc = np.clip(0.0, lg - E, lg + E)
    dmax = sig(zc) * (1 - sig(zc))
    s64, s_hi = sig(lg), sig(lg + E)
    wh = wshi[:, None]
    per = dw * s_hi + wh * (dmax * E + SIG_REL * s_hi) + U * wh * s_hi
    rgb64, B, H = np.zeros((N, 3)), np.zeros((N, 3)), np.zeros((N, 3))
    np.add.at(rgb64, srid, ws64[:, None] * s64)
    np.add.at(B, srid, per)
    np.add.at(H, srid, wh * s_hi)
    n_c = np.bincount(srid, minlength=N)[:, None]
    bg = float(kw['bg'])
    rgb64 += T64[:, None] * bg
    B += np.maximum(n_c - 1, 0) * U * H + bg * dT[:, None] + U * T_hi[:, None] * bg + U * (H + T_hi[:, None] * bg)
    # depth
    if st['kind'] == 'dcvgo':
        sd = trace['s'].double().numpy()
        dsd = 8 * U * np.ones_like(sd)
    else:
        n_samples = N_samples_of(st, kw)
        sd = (trace['step_id'].double().numpy() + 0.5) / n_samples
        dsd = 2.01 * U * sd
    depth64, BD, HD = np.zeros(N), np.zeros(N), np.zeros(N)
    np.add.at(depth64, srid, ws64 * sd)
    np.add.at(BD, srid, dw[:, 0] * (sd + dsd) + wshi * dsd + U * wshi * (sd + dsd))
    np.add.at(HD, srid, wshi * (sd + dsd))
    BD += np.maximum(n_c[:, 0] - 1, 0) * U * HD
    inf = np.zeros(N, bool)
    inf[list(skip_rays)] = True
    B[inf], BD[inf], dT[inf] = np.inf, np.inf, np.inf
    return dict(rgb=rgb64, B=B * (1 + 1e-9) + 1e-30, depth=depth64, BD=BD * (1 + 1e-9) + 1e-30, T=T64, BT=dT + 1e-30,
                w_hi=w_hi, si=si, n_c=n_c[:, 0])


def N_samples_of(st, kw):
    if st['kind'] == 'dmpigo':
        return int((st['mpi_depth'] - 1) / kw['stepsize']) + 1
    return int((st['max_world_size'] - 1) / kw['stepsize']) + 1


def check_values(out, ref64, label, ratios):
    for key, got, want, bnd in (('rgb', out['rgb_marched'].double().numpy(), ref64['rgb'], ref64['B']),
                                ('depth', out['depth'].double().numpy(), ref64['depth'], ref64['BD']),
                                ('alphainv_last', out['alphainv_last'].double().numpy(), ref64['T'], ref64['BT'])):
        err = np.abs(got - want)
        ok = err <= bnd
        assert ok.all(), (label, key, 'rays', np.nonzero(~ok)[0][:10].tolist(), float((err / bnd).max()))
        fin = np.isfinite(bnd)
        ratios['fp32 vs fp64 ' + key] = float((err[fin] / bnd[fin]).max()) if fin.any() else 0.0


def tc_bounds(st, trace, ref64, rgb_f, modes):
    """{mode: [N, 3]}: check_per_ray_against_fp32's bound on |rgb_mode - rgb_fp32| per ray, with the weights
    bounded by the recomposition's w_hi; rgb_f is fp32 mode's colour."""
    shp = types_ns(st)
    x = trace['rgb_feat'].double().numpy()
    diff = None if trace['diffuse'] is None else trace['diffuse'].double().numpy()
    D0 = FEAT_REL * np.abs(x) + 2.0 ** -24
    l_f, E_f = true_logit_bound('fp32', shp, x, diff, D0)
    w = ref64['w_hi'][ref64['si']][:, None]
    rid = trace['ray_id'].long().numpy()
    N = rgb_f.shape[0]
    bounds = {}
    for mode in modes:
        l_m, E_m = true_logit_bound(mode, shp, x, diff, D0)
        Em = np.maximum(E_m, E_f)
        zc = np.clip(0.0, l_f - Em, l_f + Em)
        dmax = sig(zc) * (1 - sig(zc))
        s_hi = sig(l_f + Em)
        per = w * (dmax * (E_m + E_f) + (2 * SIG_REL + 2 * U) * s_hi)
        B, H = np.zeros((N, 3)), np.zeros((N, 3))
        np.add.at(B, rid, per)
        np.add.at(H, rid, w * s_hi)
        bounds[mode] = B + 2 * np.maximum(ref64['n_c'][:, None] - 1, 0) * U * H + 2 * U * np.abs(rgb_f)
    return bounds


def check_tc_against_fp32(fp, outs, st, trace, ref64, skip_rays, label, ratios):
    """check_per_ray_against_fp32's bound (tc_bounds)."""
    if st['rgbnet'] is None:
        return
    N = fp['rgb_marched'].shape[0]
    keep = np.ones(N, bool)
    keep[list(skip_rays)] = False
    rgb_f = fp['rgb_marched'].double().numpy()
    bounds = tc_bounds(st, trace, ref64, rgb_f, sorted({'ws' if k[1] == 'auto' else k[1] for k in outs}))
    for k, o in outs.items():
        mode = 'ws' if k[1] == 'auto' else k[1]
        B = bounds[mode]
        d = np.abs(o['rgb_marched'].double().numpy() - rgb_f)
        ok = d[keep] <= B[keep]
        assert ok.all(), (label, k, int((~ok).sum()), float((d[keep] / np.maximum(B[keep], 1e-300)).max()))
        r = float((d[keep] / np.maximum(B[keep], 1e-300)).max()) if keep.any() else 0.0
        ratios[mode + ' vs fp32'] = max(ratios.get(mode + ' vs fp32', 0.0), r)


def run_case(st, ms, rays, kw, label, ref_ops=None):
    """One render of a scene against the oracle in every mode, order and skip setting.  Returns (fp32 output, oracle
    output, trace, borderline rays)."""
    ro, rd, vd, hw = rays[:4]
    N = ro.shape[0]
    trace, stats = {}, {}
    ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, trace=trace, **kw)
    outs = render_all(ms, ro, rd, vd, kw, hw, modes_of(st))
    base = check_modes_agree(outs, hw, float(kw['bg']), label)
    bad = set(check_geometry(base, ref, trace, st, N, label))
    if ref_ops is not None:
        dev = ms[True].density.grid.device
        tr2 = {}
        ref2 = pipeline.forward(pipeline.state_to(st, dev), ro.to(dev), rd.to(dev), vd.to(dev), ref_ops, stats={},
                                trace=tr2, **kw)
        ref2 = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in ref2.items()}
        tr2 = {k: ({n: t.cpu() for n, t in v.items()} if isinstance(v, dict) else v.cpu() if torch.is_tensor(v) else v)
               for k, v in tr2.items()}
        bad |= set(check_geometry(base, ref2, tr2, st, N, (label, 'RefExtOps')))
    ref64 = fp64_reference(st, trace, N, kw, bad)
    ratios = {}
    check_values(base, ref64, label, ratios)
    tc_outs = {k: o for k, o in outs.items() if k[1] != 'fp32'}
    check_tc_against_fp32(base, tc_outs, st, trace, ref64, bad, label, ratios)
    for k, v in ratios.items():
        RATIOS[k] = max(RATIOS.get(k, 0.0), v)
    print(f'[{label}] rays {N}  S_m/S_d/S_c {[stats[k] for k in ("S_m", "S_d", "S_c")]}  borderline {sorted(bad)}  '
          f'largest error/bound: this scene {{{", ".join(f"{k}: {v:.3g}" for k, v in ratios.items())}}}  '
          f'all scenes so far {{{", ".join(f"{k}: {v:.3g}" for k, v in RATIOS.items())}}}')
    return base, ref, trace, bad


def check_modes_agree(outs, hw, bg, label):
    """Every mode marches the same arithmetic: geometry, transmittance and depth are identical in every mode, order and
    skip setting.  fp32 colours are identical too.  A tensor-core mode computes every sample's colour independently of
    its batch, but adds a ray's samples in an order that depends on which samples share a batch (the wgmma kernels
    through shared-memory atomics, the mma.sync context per flushed group), and skipping and the tile order change the
    batches: across skip settings and orders its colours may differ only by that reassociation (order_bound).  Returns
    the fp32 render with skipping in the order hw."""
    base = outs[(True, 'fp32', hw)]
    for key, o in outs.items():
        for k in ('ray_stats', 't_minmax', 'alphainv_last', 'depth'):
            assert torch.equal(o[k], base[k]), (label, key, k)
        assert torch.equal(o['counters'][:3], base['counters'][:3]), (label, key)
        ref_o = outs[(True, key[1], hw)]
        if key[1] == 'fp32':
            assert torch.equal(o['rgb_marched'], ref_o['rgb_marched']), (label, key)
        else:
            d = (o['rgb_marched'].double() - ref_o['rgb_marched'].double()).abs()
            b = order_bound(ref_o, bg)
            assert bool((d <= b).all()), (label, key, int((d > b).sum()), float((d / b).max()))
    return base


def order_bound(out, bg):
    """|a - b| per ray for two sums of the same n terms w * sigma in different orders: each within (n - 1) u sum w sigma
    of the exact sum, plus the rounding of the background add in each.  sum w sigma comes from the colour minus its
    background, inflated by the rounding of that difference."""
    T = out['alphainv_last'].double()[:, None]
    rgb = out['rgb_marched'].double()
    s = (rgb - T * bg).abs() * (1 + 2 * U) + 2 * U * rgb.abs()
    n = out['ray_stats'][:, 3].double()[:, None]
    return 2 * (n - 1).clamp(min=0) * U * s + 2 * U * rgb.abs() + 1e-30


def shaded_per_ray(trace, N):
    return torch.bincount(trace['ray_id'].cpu().long(), minlength=N)


# ---------------------------------------------------------------------------------------------------------------------
# DirectVoxGO: off-centre, non-cubic box, anisotropic grid
# ---------------------------------------------------------------------------------------------------------------------
DIMS_A = (41, 39, 25)


@pytest.mark.parametrize('regime,thres', [('fog', 1e-4), ('fog', 0.0), ('shell', 0.05), ('blobs', 1e-4)])
def test_dvgo_offcentre_box(cuda_device, monkeypatch, regime, thres):
    st = dvgo_scene(BOX_A, DIMS_A, regime, thres)
    ms = models(st, cuda_device, monkeypatch)
    ref_ops = ref_ext_ops('dvgo', monkeypatch)
    base = dict(scenes.RENDER_KW_DVGO, bg=0.37)
    lab = f'dvgo-A-{regime}-thres{thres}'
    # orbit camera, stepsize 0.1; `far` ends before the box does: DirectVoxGO replaces it by 1e9 (lib/dvgo.py:307), so the
    # rays must not be cut there (the clamp itself is met by the 'far' edge ray below)
    out, ref, tr, _ = run_case(st, ms, orbit(24, 32), dict(base, far=3.0, stepsize=0.1), lab + '-orbit', ref_ops)
    n_c = shaded_per_ray(tr, 768)
    assert int(n_c.sum()) > 500
    if regime == 'fog':
        assert int(n_c.max()) > 384, int(n_c.max())             # a ray's samples span more than one 384-row ring
        c = tr['composited']
        assert bool((c['alpha'] == 1.0).any()) and bool((c['alpha'] == 0.0).any()) == (thres == 0)   # saturating, dead
    # camera inside the box, near 0.1
    cam = orbit(16, 24, radius=0.25)
    assert all(BOX_A[0][a] < float(cam[0][0, a]) < BOX_A[1][a] for a in range(3))
    out, ref, tr, _ = run_case(st, ms, cam, dict(base, near=0.1, stepsize=0.05), lab + '-inside', ref_ops)
    assert int(shaded_per_ray(tr, 384).sum()) > (3000 if regime != 'shell' else -1)
    # edge rays
    ro, rd, vd, hw, idx, ties = edge_rays(st)
    out, ref, tr, _ = run_case(st, ms, (ro, rd, vd, hw), dict(base, near=0.1), lab + '-edges', ref_ops)
    assert float(out['t_minmax'][idx['far'][0], 0]) == 1e9
    assert float(out['t_minmax'][idx['face'][0], 0]) == float(np.float32(BOX_A[1][0])) and int(out['ray_stats'][idx['face'][0], 1]) > 0
    # near beyond the box: one step per ray
    out, ref, tr, _ = run_case(st, ms, orbit(8, 8), dict(base, near=50.0), lab + '-near50', ref_ops)
    assert bool((out['ray_stats'][:, 0] == 1).all()) and int(out['ray_stats'][:, 1].sum()) == 0


# ---------------------------------------------------------------------------------------------------------------------
# occupancy mask of its own resolution; mask half-voxel ties
# ---------------------------------------------------------------------------------------------------------------------
DIMS_B = (42, 37, 29)
MASKS = {'coarser': (33, 29, 23), 'finer': (65, 57, 45)}      # scale 16 / 32 on every axis of BOX_B


@pytest.mark.parametrize('which', ['coarser', 'finer'])
def test_dvgo_mask_resolution_differs(cuda_device, monkeypatch, which):
    st = dvgo_scene(BOX_B, DIMS_B, 'fog', 1e-4, mask_dims=MASKS[which])
    mask = st['mask_cache']['mask']
    ro, rd, vd, hw, idx, ties = edge_rays(st)
    assert all(t is not None for t in ties)
    # each tie ray runs along a line of mask voxels at k on its two constant axes (rintf) or at k + 1 (roundf): make the
    # two lines disagree
    ks = [2 * (m // 4) for m in mask.shape]
    mask[:, ks[1], ks[2]] = False
    mask[:, ks[1] + 1, ks[2] + 1] = True
    mask[ks[0], :, ks[2]] = False
    mask[ks[0] + 1, :, ks[2] + 1] = True
    mask[ks[0], ks[1], :] = False
    mask[ks[0] + 1, ks[1] + 1, :] = True
    ms = models(st, cuda_device, monkeypatch)
    m = ms[True]
    assert tuple(m.mask_cache.mask.shape) == MASKS[which] != tuple(m.density.grid.shape[2:])
    assert torch.equal(m.mask_cache.xyz2ijk_scale.cpu(), st['mask_cache']['xyz2ijk_scale'])
    assert torch.equal(m.mask_cache.xyz2ijk_shift.cpu(), st['mask_cache']['xyz2ijk_shift'])
    ref_ops = ref_ext_ops('dvgo', monkeypatch)
    kw = dict(scenes.RENDER_KW_DVGO, bg=0.37, near=0.1)
    out, ref, tr, _ = run_case(st, ms, (ro, rd, vd, hw), kw, f'dvgo-mask-{which}-edges', ref_ops)
    for r in idx['tie']:
        assert int(out['ray_stats'][r, 1]) > 0 and int(out['ray_stats'][r, 2]) > 0, (r, out['ray_stats'][r].tolist())
    orb = orbit(32, 40)
    kw = dict(scenes.RENDER_KW_DVGO, bg=0.37)
    run_case(st, ms, orb, kw, f'dvgo-mask-{which}-orbit', ref_ops)
    f = check_skip_field(m, mask)
    assert int(f.max()) >= 3 and int(skip_reach(st, orb[0], orb[1], kw, f)) > 1000


@pytest.mark.parametrize('which', ['coarser', 'finer'])
def test_mpi_asymmetric_box_and_mask_resolution(cuda_device, monkeypatch, which):
    st = mpi_scene('fog', mask_dims={'coarser': (33, 29, 19), 'finer': (61, 53, 37)}[which])
    ms = models(st, cuda_device, monkeypatch)
    assert tuple(ms[True].mask_cache.mask.shape) != tuple(ms[True].density.grid.shape[2:])
    kw = dict(scenes.RENDER_KW_MPI, bg=0.37)
    ro, rd, vd = scenes.llff_rays(30, 40)
    out, ref, tr, _ = run_case(st, ms, (ro, rd, vd, (30, 40)), kw, f'mpi-mask-{which}', ref_ext_ops('dmpigo', monkeypatch))
    assert int(shaded_per_ray(tr, 1200).sum()) > 200
    f = check_skip_field(ms[True], st['mask_cache']['mask'])
    assert int(f.max()) >= 3 and int(skip_reach(st, ro, rd, kw, f)) > 1000


@pytest.mark.parametrize('regime', ['fog', 'shell'])
def test_mpi_asymmetric_box(cuda_device, monkeypatch, regime):
    st = mpi_scene(regime)
    ms = models(st, cuda_device, monkeypatch)
    ro, rd, vd = scenes.llff_rays(30, 40, shift=(0.11, -0.07, 0.0))
    out, ref, tr, _ = run_case(st, ms, (ro, rd, vd, (30, 40)), dict(scenes.RENDER_KW_MPI, bg=0.37), f'mpi-{regime}',
                               ref_ext_ops('dmpigo', monkeypatch))
    assert int(shaded_per_ray(tr, 1200).sum()) > 500


# ---------------------------------------------------------------------------------------------------------------------
# DirectContractedVoxGO: off-centre, anisotropic foreground box
# ---------------------------------------------------------------------------------------------------------------------
def exact_norm_rays(origin, n=1024):
    """Rays from one origin along integer directions (a, b, c) with a^2 + b^2 + c^2 a perfect square (a Pythagorean
    quadruple): every way of summing the squares is exact and so is the square root, so the marcher's direction norm
    (l2norm3_aten, an FMA chain) and the CPU's torch.norm agree bit for bit and the two front-ends see the same ray."""
    dirs = set()
    for a in range(25):
        for b in range(a, 25):
            for c in range(b, 25):
                q = a * a + b * b + c * c
                if q and math.isqrt(q) ** 2 == q and math.gcd(math.gcd(a, b), c) == 1:
                    for p in itertools.permutations((a, b, c)):
                        for sg in itertools.product((1, -1), repeat=3):
                            dirs.add(tuple(x * y for x, y in zip(p, sg)))
    dirs = sorted(dirs, key=lambda v: (sum(x * x for x in v), v))[:n]
    rd = torch.tensor(dirs, dtype=torch.float32)
    ro = torch.tensor(origin, dtype=torch.float32).expand(n, 3).contiguous()
    return ro, rd, rd / rd.norm(dim=-1, keepdim=True), (n // 32, 32)


@pytest.mark.parametrize('camera', ['outside', 'inside'])
def test_dcvgo_offcentre_foreground(cuda_device, monkeypatch, camera):
    st = dcvgo_scene('fog')
    assert len(set(st['scene_radius'].tolist())) == 3 and bool((st['scene_center'] != 0).all())
    ms = models(st, cuda_device, monkeypatch)
    assert ms[True].resolve_mlp_mode('auto') == 'ws'
    origin = (0.25, -2.5, 3.125) if camera == 'outside' else (0.125, -0.25, 0.375)
    inside = all(FG_BOX[0][a] < origin[a] < FG_BOX[1][a] for a in range(3))
    assert inside == (camera == 'inside')
    rays = exact_norm_rays(origin)
    kw = dict(scenes.RENDER_KW_DCVGO, bg=0.37)
    ref_ops = ref_ext_ops('dcvgo', monkeypatch)
    out, ref, tr, _ = run_case(st, ms, rays, kw, f'dcvgo-{camera}', ref_ops)
    assert int(shaded_per_ray(tr, 1024).sum()) > 3000
    # contracted sampling has no `far` (lib/dcvgo.py:226-262 samples a fixed t list): one well inside the foreground box
    # must change nothing
    out2, _, _, _ = run_case(st, ms, rays, dict(kw, far=0.3), f'dcvgo-{camera}-far0.3', ref_ops)
    for k in ('rgb_marched', 'alphainv_last', 'depth', 'ray_stats'):
        assert torch.equal(out2[k], out[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# a model scaled past 256^3 keeps its coarser mask (k4nerf/maintain.py, as the reference)
# ---------------------------------------------------------------------------------------------------------------------
def test_scale_volume_grid_past_256_cubed_keeps_the_mask(cuda_device, monkeypatch):
    dev = cuda_device
    st = pipeline.dvgo_state(*BOX_A, num_voxels=_num_voxels(BOX_A, DIMS_A), num_voxels_base=_num_voxels(BOX_A, DIMS_A),
                             alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=0)
    st.update(_num_voxels=_num_voxels(BOX_A, DIMS_A), _num_voxels_base=_num_voxels(BOX_A, DIMS_A), _alpha_init=1e-2)
    scenes.fill_grids(st, 'shell')
    m = model_from_state(st, dev)
    mask0 = m.mask_cache.mask.clone()
    m.scale_volume_grid(260 ** 3)                       # world size 312 x 295 x 191: 17.6 M voxels
    ws = list(m.density.grid.shape[2:])
    assert int(np.prod(ws)) > 256 ** 3 and torch.equal(m.mask_cache.mask, mask0)
    s2 = dict(st)
    s2['density'] = m.density.grid.detach().cpu()
    s2['k0'] = m.k0.grid.detach().cpu()
    s2['voxel_size'] = m.voxel_size.detach().cpu() if torch.is_tensor(m.voxel_size) else torch.tensor(float(m.voxel_size))
    s2['voxel_size_ratio'] = torch.tensor(float(m.voxel_size_ratio))
    s2['world_size'] = torch.tensor(ws)
    s2['max_world_size'] = torch.tensor(max(ws))
    ro, rd, vd = scenes.blender_rays(64, 64, crop=(24, 40, 24, 40))
    out, ref, tr, _ = run_case(s2, {True: m}, (ro, rd, vd, (16, 16)), dict(scenes.RENDER_KW_DVGO, bg=0.37), 'scaled-260')
    assert int(shaded_per_ray(tr, 256).sum()) > 1000
    del m
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# the skip field against scipy's chessboard distance transform
# ---------------------------------------------------------------------------------------------------------------------
def skip_field(m):
    from k4nerf import _lib
    sc = m._get_scene()
    n = 1 << 22
    buf = torch.zeros(n, dtype=torch.uint8, device=m.density.grid.device)
    cd = (C.c_int32 * 3)()
    st = _lib.lib.k4_testing_skip_field(sc.ptr, buf.data_ptr(), n, cd)
    if st != 0:
        return st, None
    return 0, buf[:cd[0] * cd[1] * cd[2]].cpu().numpy().reshape(tuple(cd))


def expected_field(mask):
    from scipy import ndimage
    mk = mask.cpu().numpy().astype(bool)
    c = [(s + 3) // 4 for s in mk.shape]
    pad = np.zeros([4 * x for x in c], bool)
    pad[:mk.shape[0], :mk.shape[1], :mk.shape[2]] = mk
    occ = pad.reshape(c[0], 4, c[1], 4, c[2], 4).any(axis=(1, 3, 5))
    if not occ.any():
        return np.full(c, 49, np.uint8)
    return np.minimum(ndimage.distance_transform_cdt(~occ, metric='chessboard'), 49).astype(np.uint8)


def check_skip_field(m, mask):
    st, f = skip_field(m)
    assert st == 0, st
    want = expected_field(mask)
    assert f.shape == want.shape and np.array_equal(f, want), (f.shape, want.shape, int((f != want).sum()))
    return f


def skip_reach(st, ro, rd, kw, field):
    """In-box samples of the oracle's sampler that land in a skip cell at distance >= 3: a marcher there may jump over
    the rest of a (5 x 4)^3-voxel empty region.  Skipping is count-preserving -- the skipped samples are added to S_m --
    so renders with and without it are equal by contract; this count shows that the scenes give it long jumps to make."""
    mc = st['mask_cache']
    if st['kind'] == 'dmpigo':
        n = int((st['mpi_depth'] - 1) / kw['stepsize']) + 1
        pts, out = ops.CpuOps.sample_ndc_pts_on_rays(ro, rd, st['xyz_min'], st['xyz_max'], n)
    else:
        pts, out = ops.CpuOps.sample_pts_on_rays(ro, rd, st['xyz_min'], st['xyz_max'], kw['near'], 1e9,
                                                 float(kw['stepsize'] * st['voxel_size']))[:2]
    p = pts.reshape(-1, 3)[~out.reshape(-1)].double().numpy()
    x = p * mc['xyz2ijk_scale'].double().numpy() + mc['xyz2ijk_shift'].double().numpy()
    idx = (np.sign(x) * np.floor(np.abs(x) + 0.5)).astype(np.int64)
    ms = np.array(mc['mask'].shape)
    inside = ((idx >= 0) & (idx < ms)).all(1)
    c = idx[inside] // 4
    return int((field[c[:, 0], c[:, 1], c[:, 2]] >= 3).sum())


def _mask_model(dev, mdims, occupied):
    st = pipeline.dvgo_state(*BOX_B, num_voxels=8 * 7 * 6, num_voxels_base=8 * 7 * 6, alpha_init=1e-2,
                             fast_color_thres=1e-4, rgbnet_dim=0, mask_cache_world_size=list(mdims))
    st.update(_num_voxels=8 * 7 * 6, _num_voxels_base=8 * 7 * 6, _alpha_init=1e-2)
    mask = torch.zeros(mdims, dtype=torch.bool)
    for i, j, k in occupied:
        mask[i, j, k] = True
    st['mask_cache'] = pipeline.mask_grid_state(mask, st['xyz_min'], st['xyz_max'])
    return model_from_state(st, dev), mask


@pytest.mark.parametrize('mdims,occupied', [
    ((5, 5, 5), [(2, 2, 2)]),
    ((5, 9, 13), [(4, 0, 12)]),
    ((17, 21, 9), [(0, 0, 0), (16, 20, 8)]),
    ((13, 5, 17), []),                                    # nothing occupied: the cap everywhere
    ((205, 6, 5), [(0, 5, 0)]),                           # 52 cells along x: the true distances pass the cap
    ((9, 201, 7), [(8, 200, 6), (4, 3, 2)]),
])
def test_skip_field_equals_chessboard_transform(cuda_device, mdims, occupied):
    m, mask = _mask_model(cuda_device, mdims, occupied)
    f = check_skip_field(m, mask)
    if max(mdims) > 200 and len(occupied) == 1:
        assert int(f.max()) == 49 and int((f == 48).sum()) > 0


def test_skip_field_absent(cuda_device, monkeypatch):
    """No field where skipping is off: K4_NO_SKIP, a mask axis of one voxel (scale 0: every point maps to voxel 0, the
    skip geometry needs 1 / scale), and DirectContractedVoxGO."""
    m, _ = _mask_model(cuda_device, (5, 1, 9), [(2, 0, 3)])
    assert skip_field(m)[0] == -2
    monkeypatch.setenv('K4_NO_SKIP', '1')
    m, _ = _mask_model(cuda_device, (5, 5, 9), [(2, 0, 3)])
    assert skip_field(m)[0] == -2
    monkeypatch.delenv('K4_NO_SKIP')
    m = model_from_state(dcvgo_scene('fog'), cuda_device)
    assert skip_field(m)[0] == -2


# ---------------------------------------------------------------------------------------------------------------------
# occupancy maintenance with a mask of its own resolution
# ---------------------------------------------------------------------------------------------------------------------
def _torch_alpha(den, shift, interval):
    return 1 - torch.pow(1 + torch.exp(den + shift), -interval)


@pytest.mark.parametrize('kind', ['dvgo', 'mpi'])
def test_update_occupancy_cache_with_own_mask_resolution(cuda_device, kind):
    dev = cuda_device
    if kind == 'dvgo':
        st = dvgo_scene(BOX_A, DIMS_A, 'fog', 1e-4, mask_dims=(23, 53, 19))
    else:
        st = mpi_scene('fog', mask_dims=(61, 29, 37))
    st['mask_cache']['mask'] = torch.ones_like(st['mask_cache']['mask'])
    m = model_from_state(st, dev)
    with torch.no_grad():
        if kind == 'mpi':
            m.density.grid.sub_(8.0)
        else:
            m.density.grid.clamp_(-30, 30).mul_(4.0).sub_(2.0)
    mask0 = m.mask_cache.mask.clone()
    shp = mask0.shape
    assert tuple(shp) != tuple(m.density.grid.shape[2:])
    xyz = torch.stack(torch.meshgrid(*[torch.linspace(float(m.xyz_min[a]), float(m.xyz_max[a]), shp[a], device=dev)
                                       for a in range(3)], indexing='ij'), -1)
    ind = ((xyz.reshape(1, 1, 1, -1, 3) - m.xyz_min) / (m.xyz_max - m.xyz_min)).flip((-1,)) * 2 - 1
    den = F.grid_sample(m.density.grid, ind, mode='bilinear', align_corners=True).reshape(shp)
    shift = 0.0 if kind == 'mpi' else float(m.act_shift)
    alpha = _torch_alpha(den, shift, float(m.voxel_size_ratio))
    thres = float(torch.quantile(alpha.detach().flatten(), 0.985))
    assert 0 < thres < 0.999
    m.fast_color_thres = thres
    want = mask0 & (F.max_pool3d(alpha[None, None], kernel_size=3, padding=1, stride=1)[0, 0] > thres)
    m.update_occupancy_cache()
    got = m.mask_cache.mask
    assert got.shape == shp
    flips = int((got != want).sum())
    assert flips <= max(1, int(1e-4 * got.numel())), (flips, got.numel())
    assert 0 < int(got.sum()) < got.numel()
