"""GPU: the fused training step (k4nerf.train_fused.render_loss, csrc/k4_train_march.cu) against the float64 autograd
restatement of train_ref64.py with run_sr.py's composite loss (nearclip 0), and against the materialised path.

The bounds are train_ref64.Bounds (the error model of test_gpu_train_grad.py's docstring) plus the error term the fused
arithmetic adds, derived here (u = 2^-24, v = 2^-53; n_r the ray's composited samples, sums over its shaded samples k):
  * B_i, the suffix sum of Alphas2Weights.backward, is the forward's per-ray total minus the backward's running prefix,
    both fp64 sums of at most n_r terms (the distortion gradient's W>i, WM>i likewise).  Every partial sum is at most
    M_r = sum_k |dL/dw_k| w_k + |g_rgbm| . rgb_feature + cd (8 W_r^2 + 2/3 I sum w^2)
    (|dL/dw_k| <= |g_rgbm| . c_k + cd (4 W_r + I w_k), W_r = sum w, s <= 1, so pair <= 2 W_r^2), so B_i is off by at most
    E_B = (4 n_r + 16) v M_r before its one rounding to fp32, which the restatement's own (n_r + 2) u bound covers.
  * the kernel divides B_i by fp32(1 - alpha_i) + 1e-10, not by the exact 1 - alpha_i: for a near-opaque sample whose
    alpha rounds to 1 that is 1e-10.  The denominator is at least max(1 - alpha_i - E_alpha_i - u, 0) + 1e-10
    (E_alpha: Bounds.alpha_occ), so dL/dalpha_i moves by E_B / that, and dL/dx_i by alpha'(x_i) times that; the density
    grid's bound takes the scatter of this term with the trilinear weights.  (With the suffix in fp32 instead, the
    residual of the empty suffix behind a ray's last sample, a few ulp of the total, came out of that division as a
    10-30 % error on the voxels of such samples.)  k0 and rgbnet gradients take no suffix: their bounds are Bounds' own.
  * loss terms: each term's first-order sensitivity to the per-ray / per-sample bounds of Bounds (rgb_marched,
    alphainv_last, weights, raw_rgb), the fp32 per-ray sums ((n_r + 6) u of their absolute terms), and 4u for the fp64
    reduction's final rounding.
Each case prints its largest observed error as a fraction of its bound.
"""
import math

import pytest
import torch

import train_ref64 as R
from test_gpu_train_grad import CASES, Ratio, _model, build_case, no_tf32  # noqa: F401  (fixture)
from helpers import make_state
from oracle import scenes

pytestmark = pytest.mark.gpu

U = R.U
FULL = dict(main=1.0, entropy_last=0.01, distortion=0.01, rgbper=0.1)
FUSED_CASES = [c for c in CASES if not c.startswith('dcvgo')]


def _lw(kind, lw):
    return dict(lw, distortion=0.0) if kind == 'dvgo' else dict(lw)


def _names(m):
    from k4nerf._scene import linear_layers
    names = {id(p): k for k, p in m.named_parameters()}
    lin = {}
    for i, l in enumerate(linear_layers(m.rgbnet)):
        lin[names[id(l.weight)]], lin[names[id(l.bias)]] = f'rgbnet.L{i}.weight', f'rgbnet.L{i}.bias'
    return lin


def _grads(m):
    lin = _names(m)
    return {lin.get(k, k): p.grad for k, p in m.named_parameters() if p.grad is not None}


def run_fused(m, ro, rd, vd, target, kw, lw, dev):
    from k4nerf import train_fused
    torch.cuda.manual_seed(1234)
    loss, out = train_fused.render_loss(m, ro.to(dev), rd.to(dev), vd.to(dev), target.to(dev), 1, kw, loss_weights=lw)
    loss.backward()
    torch.cuda.synchronize()
    return loss, out


def reference(P, ro, rd, vd, target, kw, lw, dev):
    def rand_bkgd(shape):
        torch.cuda.manual_seed(1234)
        return torch.rand(shape, device=dev, dtype=torch.float32).cpu()
    n = ro.shape[0]
    ref = R.forward64(P, ro, rd, vd, kw, global_step=1, is_train=True, rand_bkgd=rand_bkgd, sample_device=dev)
    lw64 = dict(lw, nearclip=0.0)
    R.composite_loss(ref, target, n, weights=lw64).backward()
    b = R.Bounds(P, ref, target, n, lw=lw64)
    bad = R.check_margins(P, b, ref)
    assert not bad, ('borderline sample: fp32 and fp64 may take it to different fates', bad)
    return ref, b


def fused_extra(P, ref, b, target, lw):
    """The density-grid bound's extra term of the fused arithmetic (module docstring), flat [X*Y*Z]."""
    st = ref['_']
    n = target.shape[0]
    tgt = target.double()
    rid2, w2, rgb = ref['ray_id'], ref['weights'].detach(), ref['raw_rgb'].detach()
    g_rgbm = 2 * lw['main'] / (3 * n) * (ref['rgb_marched'].detach() - tgt)
    Wr = torch.zeros(n, dtype=torch.float64).index_add_(0, rid2, w2)
    Q = torch.zeros(n, dtype=torch.float64).index_add_(0, rid2, w2 * w2)
    rgbf = torch.zeros(n, 3, dtype=torch.float64).index_add_(0, rid2, w2[:, None] * rgb)
    cd, Id = 0.0, 0.0
    if lw['distortion'] > 0 and P['kind'] != 'dvgo' and rid2.numel():
        cd, Id = lw['distortion'] / (int(rid2.max()) + 1), 1.0 / ref['n_max']
    gw_abs = (g_rgbm[rid2].abs() * rgb).sum(1) + cd * (4 * Wr[rid2] + Id * w2)
    M = torch.zeros(n, dtype=torch.float64).index_add_(0, rid2, gw_abs * w2) + (g_rgbm.abs() * rgbf).sum(1) + \
        cd * (8 * Wr ** 2 + (2 / 3) * Id * Q)
    E_B = (4 * b.n_r + 16) * 2.0 ** -53 * M
    rid1, live = st['comp_ray_id'], st['comp_live']
    x, I = st['x'], st['interval']
    p = torch.exp(-I * torch.nn.functional.softplus(x))
    sel = st['sel_alpha']
    den = (p[sel] - b.alpha_occ[sel] - U).clamp_min(0) + 1e-10
    ea = E_B[rid1] / den * live
    ea0 = torch.zeros_like(x).masked_scatter_(sel, ea)
    ex = I * torch.sigmoid(x) * p * ea0
    X, Y, Z = P['density'].shape[2:]
    idx, wc = R.corners(st['occ_pts'], P['xyz_min'], P['xyz_max'], (X, Y, Z))
    return R.scatter_corners(wc * ex[:, None], idx, X * Y * Z)


def term_refs(P, ref, b, target, lw):
    """(value, bound) of each weighted loss term in fp64."""
    n = target.shape[0]
    tgt = target.double()
    rgbm, E_m = ref['rgb_marched'].detach(), b.rgb_marched
    T, E_T = ref['alphainv_last'].detach(), b.alphainv_last
    rid2, w2, E_w = ref['ray_id'], ref['weights'].detach(), b.weights
    rgb, E_c = ref['raw_rgb'].detach(), b.raw_rgb
    nmax = int(b.n_r.max()) if b.n_r.numel() else 0
    out = {}
    d = rgbm - tgt
    v = lw['main'] * (d * d).sum() / (3 * n)
    out['loss_main'] = (v, lw['main'] * (2 * d.abs() * E_m + E_m * E_m).sum() / (3 * n) + 4 * U * v)

    def ent(q):
        q = q.clamp(1e-6, 1 - 1e-6)
        return -(q * torch.log(q) + (1 - q) * torch.log(1 - q))
    v = lw['entropy_last'] * ent(T).sum() / n
    lo, hi = (T - E_T), (T + E_T)
    dev_ = torch.maximum((ent(lo) - ent(T)).abs(), (ent(hi) - ent(T)).abs())
    dev_ = torch.where((lo < 0.5) & (hi > 0.5), torch.maximum(dev_, (ent(torch.full_like(T, 0.5)) - ent(T)).abs()), dev_)
    out['loss_entropy_last'] = (v, lw['entropy_last'] * dev_.sum() / n + 4 * U * v)
    v = torch.zeros((), dtype=torch.float64)
    bd = torch.zeros((), dtype=torch.float64)
    if lw['distortion'] > 0 and P['kind'] != 'dvgo' and rid2.numel():
        v = lw['distortion'] * R.flatten_eff_distloss(w2, ref['s'].detach().double(), 1 / ref['n_max'], rid2)
        cd, Id = lw['distortion'] / (int(rid2.max()) + 1), 1.0 / ref['n_max']
        Wr = torch.zeros(n, dtype=torch.float64).index_add_(0, rid2, w2)
        Q = torch.zeros(n, dtype=torch.float64).index_add_(0, rid2, w2 * w2)
        Ew_r = torch.zeros(n, dtype=torch.float64).index_add_(0, rid2, E_w)
        bd = (cd * (4 * Wr[rid2] + Id * w2) * E_w).sum() + cd * (2 * Ew_r ** 2).sum() + \
            cd * ((2 * b.n_r + 8) * U * (4 * Wr ** 2 + Id * Q)).sum() + 4 * U * v
    out['loss_distortion'] = (v, bd)
    v = torch.zeros((), dtype=torch.float64)
    bd = torch.zeros((), dtype=torch.float64)
    if lw['rgbper'] > 0 and rid2.numel():
        e = rgb - tgt[rid2]
        v = lw['rgbper'] * (w2 * (e * e).sum(1)).sum() / n
        bd = lw['rgbper'] * ((E_w * (e * e).sum(1) + w2 * (2 * e.abs() * E_c + E_c * E_c).sum(1)).sum() +
                             (nmax + 6) * U * (w2 * (e * e).sum(1)).sum()) / n + 4 * U * v
    out['loss_rgbper'] = (v, bd)
    return out


def compare(m, P, ref, b, out, loss, target, lw, q, scale=1.0, extra=None):
    """rgb_marched, alphainv_last, the terms, the total and every parameter gradient within scale x the bounds."""
    q.check('rgb_marched', out['rgb_marched'], ref['rgb_marched'], scale * b.rgb_marched)
    q.check('alphainv_last', out['alphainv_last'], ref['alphainv_last'], scale * b.alphainv_last)
    terms = term_refs(P, ref, b, target, lw)
    tot_v, tot_b = 0.0, 0.0
    for k, (v, bd) in terms.items():
        q.check(k, out[k].reshape(1), torch.as_tensor(v).reshape(1), torch.as_tensor(bd).reshape(1))
        tot_v, tot_b = tot_v + v, tot_b + bd
    q.check('loss', loss.detach().reshape(1), torch.as_tensor(tot_v).reshape(1),
            torch.as_tensor(tot_b + 4 * U * abs(float(tot_v))).reshape(1))
    ours = _grads(m)
    theirs = {k: p.grad for k, p in R.trainable(P).items() if p.grad is not None}
    assert set(ours) == set(theirs), (sorted(ours), sorted(theirs))
    for k in theirs:
        bound = scale * b.params[k]
        if k == 'density.grid' and extra is not None:
            bound = bound + extra
        q.check(k, ours[k], theirs[k], bound)


def run_case(cid, dev, lw=FULL, seed=0):
    st, act, ro, rd, vd, kw = build_case(cid)
    lw = _lw(st['kind'], lw)
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(seed))
    m = _model(st, act, dev)
    P = R.params_from_model(m)
    loss, out = run_fused(m, ro, rd, vd, target, kw, lw, dev)
    ref, b = reference(P, ro, rd, vd, target, kw, lw, dev)
    q = Ratio()
    compare(m, P, ref, b, out, loss, target, lw, q, extra=fused_extra(P, ref, b, target, lw))
    return q.worst


@pytest.mark.parametrize('cid', FUSED_CASES)
def test_fused_matches_float64_restatement(cuda_device, no_tf32, cid):
    worst = run_case(cid, cuda_device)
    print(f'\n[train_fused {cid}] worst observed/bound {max(worst.values()):.3g} ({max(worst, key=worst.get)})')


@pytest.mark.parametrize('term', sorted(FULL))
@pytest.mark.parametrize('cid', ['mpi_relu_pe_randbkgd_shell', 'mpi_gauss_fog', 'dvgo_nondirect_slab'])
def test_each_loss_term_alone(cuda_device, no_tf32, cid, term):
    if term == 'distortion' and cid.startswith('dvgo'):
        pytest.skip('DirectVoxGO has no distortion loss')
    lw = {k: (v if k == term else 0.0) for k, v in FULL.items()}
    worst = run_case(cid, cuda_device, lw=lw)
    print(f'\n[train_fused {cid} {term} only] worst observed/bound {max(worst.values()):.3g}')


def test_fused_against_materialised_path(cuda_device):
    """Same model and seed: the same rgb_marched (within both paths' bounds; the rand_bkgd draw is the same), gradients
    within the sum of both paths' bounds."""
    cid = 'mpi_relu_pe_randbkgd_shell'
    st, act, ro, rd, vd, kw = build_case(cid)
    n = ro.shape[0]
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(3))
    m1, m2 = _model(st, act, cuda_device), _model(st, act, cuda_device)
    P = R.params_from_model(m1)
    loss, out = run_fused(m1, ro, rd, vd, target, kw, FULL, cuda_device)
    torch.cuda.manual_seed(1234)
    o2 = m2(ro.to(cuda_device), rd.to(cuda_device), vd.to(cuda_device), global_step=1, is_train=True, **kw)
    R.composite_loss(o2, target.to(cuda_device), n, weights=dict(FULL, nearclip=0.0)).backward()
    torch.cuda.synchronize()
    ref, b = reference(P, ro, rd, vd, target, kw, FULL, cuda_device)
    q = Ratio()
    q.check('rgb_marched fused vs materialised', out['rgb_marched'], o2['rgb_marched'], 2 * b.rgb_marched)
    g1, g2 = _grads(m1), _grads(m2)
    assert set(g1) == set(g2)
    extra = fused_extra(P, ref, b, target, FULL)
    for k in g1:
        bound = 2 * b.params[k] + (extra if k == 'density.grid' else 0)
        q.check(f'{k} fused vs materialised', g1[k], g2[k], bound)
    print(f'\n[train_fused vs materialised] worst observed/bound {max(q.worst.values()):.3g}')


def test_all_miss_batch(cuda_device):
    """Every ray misses the box: every gradient is exactly zero; the loss is the main and entropy terms only."""
    st, act, ro, rd, vd, kw = build_case('mpi_relu_fog')
    ro = ro[:40].clone()
    ro[:, 0] += 50.0
    rd, vd = rd[:40].clone(), vd[:40].clone()
    m = _model(st, act, cuda_device)
    target = torch.rand(40, 3, generator=torch.Generator().manual_seed(0))
    loss, out = run_fused(m, ro, rd, vd, target, kw, FULL, cuda_device)
    assert torch.equal(out['alphainv_last'].cpu(), torch.ones(40))
    assert float(out['loss_distortion']) == 0.0 and float(out['loss_rgbper']) == 0.0
    assert float(loss) == pytest.approx(float(out['loss_main']) + float(out['loss_entropy_last']), rel=1e-6)
    g = _grads(m)
    assert set(g) == {'density.grid', 'k0.grid'} | {f'rgbnet.L{i}.{w}' for i in range(3) for w in ('weight', 'bias')}
    for k, v in g.items():
        assert torch.count_nonzero(v) == 0, k


def _mpi_case():
    st, act, ro, rd, vd, kw = build_case('mpi_gauss_fog')
    return st, act, ro, rd, vd, kw, torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(1))


def test_no_host_sync(cuda_device):
    from k4nerf import train_fused
    st, act, ro, rd, vd, kw, target = _mpi_case()
    m = _model(st, act, cuda_device)
    args = [t.to(cuda_device) for t in (ro, rd, vd, target)]
    train_fused.render_loss(m, *args[:3], args[3], 1, kw)[0].backward()       # caches the model's host constants
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss, out = train_fused.render_loss(m, *args[:3], args[3], 1, kw)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_loss_bitwise_reproducible_and_grads_accumulate(cuda_device):
    from k4nerf import train_fused
    st, act, ro, rd, vd, kw, target = _mpi_case()
    m = _model(st, act, cuda_device)
    args = [t.to(cuda_device) for t in (ro, rd, vd, target)]
    losses = []
    for _ in range(3):
        loss, out = train_fused.render_loss(m, *args[:3], args[3], 1, kw)
        losses.append(torch.cat([loss.reshape(1), out['loss_main'].reshape(1), out['loss_entropy_last'].reshape(1),
                                 out['loss_distortion'].reshape(1), out['loss_rgbper'].reshape(1)]).cpu())
    assert all(torch.equal(losses[0], x) for x in losses[1:])
    m.zero_grad(set_to_none=True)
    train_fused.render_loss(m, *args[:3], args[3], 1, kw)[0].backward()
    g1 = {k: v.clone() for k, v in _grads(m).items()}
    train_fused.render_loss(m, *args[:3], args[3], 1, kw)[0].backward()
    g2 = _grads(m)
    for k in g1:
        assert torch.equal(g2[k] == 0, g1[k] == 0), k
        torch.testing.assert_close(g2[k], 2 * g1[k], rtol=1e-5, atol=1e-7 * float(g1[k].abs().max()) + 1e-30)


def test_untouched_voxels_are_exactly_zero(cuda_device):
    st, act, ro, rd, vd, kw = build_case('dvgo_direct_shell')
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(2))
    m = _model(st, act, cuda_device)
    P = R.params_from_model(m)
    run_fused(m, ro, rd, vd, target, kw, _lw('dvgo', FULL), cuda_device)
    ref, b = reference(P, ro, rd, vd, target, kw, _lw('dvgo', FULL), cuda_device)
    g = _grads(m)
    untouched_d = b.count_density == 0
    assert untouched_d.any()
    assert torch.equal(g['density.grid'].reshape(-1).cpu()[untouched_d], torch.zeros(int(untouched_d.sum())))
    untouched_k = b.count_k0 == 0
    gk = g['k0.grid'].reshape(g['k0.grid'].shape[1], -1).cpu()
    assert torch.count_nonzero(gk[:, untouched_k]) == 0


def test_larger_mpi_case(cuda_device, no_tf32):
    """96 x 96 x 64 MPI, 2048 rays (64 CTAs), every occupied sample shaded: full 32-row weight batches in every warp and
    grid atomics from many rays.  fast_color_thres 0 and the fog shifted down by 2 keep every sample away from the alpha /
    weight thresholds and every ray short of the T < 1e-3 stop, which the margin check needs at this sample count."""
    st = make_state('cfgB', xy=96, depth=64, regime='fog', width=64)
    st['fast_color_thres'] = 0.0
    st['density'] = st['density'] - 2.0
    kw = dict(scenes.RENDER_KW_MPI)
    ro, rd, vd = scenes.llff_rays(32, 64)
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(4))
    m = _model(st, 'relu', cuda_device)
    P = R.params_from_model(m)
    loss, out = run_fused(m, ro, rd, vd, target, kw, FULL, cuda_device)
    ref, b = reference(P, ro, rd, vd, target, kw, FULL, cuda_device)
    q = Ratio()
    compare(m, P, ref, b, out, loss, target, FULL, q, extra=fused_extra(P, ref, b, target, FULL))
    assert ref['ray_id'].numel() > 100_000
    print(f'\n[train_fused large MPI] shaded {ref["ray_id"].numel()}, worst observed/bound {max(q.worst.values()):.3g}')
    assert math.isfinite(float(loss))
