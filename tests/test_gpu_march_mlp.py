"""GPU: the marchers' colour MLP (rgbnet) sample by sample, and per ray, against float64 references.

Element level: k4_testing_rgbnet runs a scene's packed rgbnet on rows the test supplies, with the device code of one MLP
mode -- mlp_batch_wgmma on a ring tile written through the scene's column map (ws), MmaWarpCtx driven as k4_march.cu
drives it (f16 / f16x3), mlp_fp32 (fp32) -- and returns what the marchers accumulate into a ray: per group of G rows
(128 for wgmma, 32 otherwise) and owner j, the sum of w * sigmoid(logit (+ diffuse)) over the rows j owns.  The models are
the 12 wgmma configurations of csrc/k4_ws_cfgs.h at their exact shapes plus the models of test_gpu_marcher.WS_SHAPES that
run zero-padded on a larger configuration; every model runs in every mode it has a build for.

Per ray: every tensor-core mode against fp32 mode on every WS_SHAPES model, and ws against fp32 mode on scenes that
stress the ring (long queues next to empty rays, one live ray per tile, more tiles than marcher groups), bounded per
sample with the weights and rgbnet inputs that oracle.pipeline.forward(trace=...) records.  This is what checks the row
assembly of the marchers themselves (k0 channels, position code, view embedding, the column map of a padded wgmma
configuration, the diffuse logits) and which ray a sample is credited to.

Error model (u = 2^-24, the unit roundoff of fp32):
  * tensor-core accumulation: every MMA instruction adds at most 16 exact fp16 products to the fp32 accumulator.  Aligned
    to the largest exponent and truncated to the fp32 significand, each of those 17 terms loses less than one ulp of the
    largest, so one instruction errs by at most 17 * 2^-23 * (|accumulator| + sum |products|) <= 17 * 2^-23 * S, with S =
    |bias| + sum |a| |w| of the layer.  A layer of n instructions: n * 17 * 2^-23 * S (K = 128: about 2^-16 * S).
  * fp32 mode: one rounded FMA per input from the bias: K * u * S.
  * f16x3: x = hi + lo with hi = fp16(x), lo = fp16(x - hi); |x - hi - lo| <= 2^-22 |x| + 2^-25 (lo may be subnormal) and
    |lo| <= 2^-11 |x| + 2^-24.  The product drops lo_x * lo_w and the two representation errors.  Its three MMAs per k
    step are each charged the accumulation error above, so the random-operand bound of f16x3 comes out a few times
    LOOSER than that of f16 (against f16's quantised reference), not tighter; it still lies far below the 2^-11-class
    error of a lost lo term, and test_f16x3_keeps_the_lo_parts_exactly checks the compensation bit for bit.
  * hidden layers of f16 / wgmma are rounded to fp16 by design: the reference rounds them too, and where the kernel's
    interval [a - E, a + E] straddles an fp16 rounding boundary the bound takes the spread of the rounded interval.
  * sigmoid_ref = 1 / (1 + expf(-x)): expf <= 2 ulp, the add and the division 1/2 ulp each: <= 3 * 2^-23 relative.
  * w * sigma: 1/2 ulp; a sum of n such terms (in any order): (n - 1) * u * sum.
"""
import ctypes as C
import types
import zlib

import numpy as np
import pytest
import torch

from helpers import make_state, model_from_state, rays_for
from march_bounds import (FEAT_REL, GAMMA_TC, SIG_REL, U, WS_CFGS, dim0_of, f16, logit_bound, shape_info, sig, supports,
                          true_logit_bound)
from test_gpu_marcher import WS_SHAPES, _blob_state

pytestmark = pytest.mark.gpu

ROWS = [1, 31, 32, 33, 63, 64, 65, 127, 128, 300]
MODES = {'fp32': 0, 'f16': 1, 'f16x3': 2, 'ws': 4}

def _models():
    """(name, kind, C, vpe, spe, width, direct, config id): the exact shapes, then the padded WS_SHAPES models."""
    out, seen = [], set()
    for cid, kind, c, vpe, spe, w, d in WS_CFGS:
        out.append((f'cfg{cid}', kind, c, vpe, spe, w, d, cid))
        seen.add((kind, c, vpe, spe, w, d))
    for kind, kw, cid in WS_SHAPES:
        key = (kind, kw['k0_dim'], kw['viewbase_pe'], kw.get('spatial_pe', 0), kw['width'], int(kw.get('rgbnet_direct', True)))
        if key not in seen:
            seen.add(key)
            out.append((f'{kind}-C{key[1]}-v{key[2]}-s{key[3]}-w{key[4]}-d{key[5]}-on{cid}', *key, cid))
    return out


MODELS = _models()
MODEL_IDS = [m[0] for m in MODELS]


class Model:
    """A scene of one rgbnet shape with the given layer weights, on the device."""

    def __init__(self, spec, layers, dev):
        name, kind, c, vpe, spe, w, direct, cid = spec
        kw = dict(k0_dim=c, viewbase_pe=vpe, width=w)
        if kind == 'cfgA':
            kw['rgbnet_direct'] = bool(direct)
            st = make_state(kind, res=8, regime='fog', **kw)
        elif kind == 'cfgB':
            st = make_state(kind, xy=8, depth=8, regime='fog', spatial_pe=spe, **kw)
        else:
            st = make_state(kind, res=8, regime='fog', **kw)
        assert [tuple(l[0].shape) for l in st['rgbnet']] == [tuple(W.shape) for W, _ in layers]
        st['rgbnet'] = [(torch.tensor(W, dtype=torch.float32), torch.tensor(b, dtype=torch.float32)) for W, b in layers]
        self.layers = [(l[0].double().numpy(), l[1].double().numpy()) for l in st['rgbnet']]     # fp32 values in fp64
        self.m = model_from_state(st, dev)
        self.spec, self.dev = spec, dev
        self.kind, self.direct, self.width, self.cid = kind, bool(direct), w, cid
        shape_info(self, spec)

    def supports(self, mode):
        return supports(self.spec, mode)

    def run(self, mode, x, diff, w, owner):
        """k4_testing_rgbnet -> (status, racc [n_groups, G, 3] float64, G)."""
        from k4nerf import _lib
        n = x.shape[0]
        t = lambda a, dt: torch.tensor(np.ascontiguousarray(a), dtype=dt, device=self.dev)
        tx, tw, to = t(x, torch.float32), t(w, torch.float32), t(owner, torch.int32)
        td = t(diff, torch.float32) if diff is not None else None
        racc = torch.full(((n + 31) // 32 * 32 * 3 + 128 * 3,), float('nan'), device=self.dev)
        a = _lib.RgbnetTestArgs()
        a.mode, a.n = MODES[mode], n
        a.d_x, a.d_w, a.d_owner, a.d_racc = tx.data_ptr(), tw.data_ptr(), to.data_ptr(), racc.data_ptr()
        a.d_diffuse = td.data_ptr() if td is not None else None
        g = C.c_int32(0)
        st = _lib.lib.k4_testing_rgbnet(self.m._get_scene().ptr, C.byref(a), C.byref(g),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert st in (0, -2), (self.spec[0], mode, st, _lib.lib.k4_last_cuda_error().decode())
        if st != 0:
            return st, None, 0
        G = g.value
        ng = (n + G - 1) // G
        return st, racc[:ng * G * 3].view(ng, G, 3).double().cpu().numpy(), G


def group_size(mode):
    return 128 if mode == 'ws' else 32


def perm_owners(n, G, rng):
    """Every row its own owner: a random permutation of [0, G) inside each group."""
    return np.concatenate([rng.permutation(G)[:min(G, n - s)] for s in range(0, n, G)]).astype(np.int32)


def per_row(racc, owner, G):
    n = owner.shape[0]
    return racc[np.arange(n) // G, owner]


def unowned_zero(racc, owner, G):
    hit = np.zeros(racc.shape[:2], bool)
    hit[np.arange(owner.shape[0]) // G, owner] = True
    return bool((racc[~hit] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# a. exact operands
# ---------------------------------------------------------------------------------------------------------------------
def exact_operands(dim0, width, direct, n, rng, lo_parts=False):
    """Operands for which every intermediate of every mode is exact, so that all modes must agree bit for bit.

    Inputs: column 0 is the constant 1/2, the others k/16 with |k| <= 8.  Layer 1: hidden unit 0 has no weights and bias
    2^-5, so h1_0 = 1/32 in every row.  Unit j >= 1 has bias b = q/128 + m 2^-14 (q in [32, 64), m = +-1): fp16(b) = q/128
    (the fp16 ulp there is 2^-12), so the wgmma bias tile holds hi = q/128 and a non-zero lo = m 2^-14.  Its weight on
    column 0 is -q/64, which cancels hi, plus two weights r/64 with |r| <= 2.  So a1 = m 2^-14 + (two products on the 2^-10
    grid), |a1| < 2^-5: a multiple of 2^-14 below 2^-3, exact in fp16; every partial sum is a multiple of 2^-14 below 1,
    exact in fp32 in any order.  Layer 2 repeats this with h1_0: weight -8 on unit 0 cancels hi = 1/4 of b = 1/4 + m 2^-14,
    plus two weights in {+-1, +-2} and {+-1}: |a2| < 2^-3 on the 2^-14 grid.  Layer 3: b = +-q/128 + m 2^-14 and four
    weights in {+-1, +-2, +-4}: |logit| < 2.5 on the 2^-14 grid, exact in fp32.  Diffuse logits k/16 add exactly; the
    weights w = 2^-e make w * sigmoid exact.

    lo_parts: inputs k/16 + j 2^-15 (|k| in [5, 8), |j| <= 3) and layer-1 weights r/64 + q 2^-18 (r = +-1, +-2, |q| <= 1)
    have non-zero fp16 lo parts, which only f16x3 keeps: its three products hi*hi + lo*hi + hi*lo are multiples of 2^-22
    and the sums stay below 2^-5 (layer 1) and 2.5 (logits), exact in fp32; the hidden values split exactly into hi + lo."""
    x = rng.integers(-8, 9, size=(n, dim0)) / 16.0
    if lo_parts:
        x = rng.choice([-1, 1], size=(n, dim0)) * rng.integers(5, 8, size=(n, dim0)) / 16.0 + rng.integers(-3, 4, size=(n, dim0)) * 2.0 ** -15
    x[:, 0] = 0.5
    W1 = np.zeros((width, dim0))
    b1 = np.zeros(width)
    b1[0] = 2.0 ** -5
    for j in range(1, width):
        q = rng.integers(32, 64)
        b1[j] = q / 128 + rng.choice([-1, 1]) * 2.0 ** -14
        W1[j, 0] = -q / 64
        for c in rng.choice(np.arange(1, dim0), size=2, replace=False):
            r = rng.choice([-2, -1, 1, 2]) if lo_parts else rng.integers(-2, 3)
            W1[j, c] = r / 64 + (rng.integers(-1, 2) * 2.0 ** -18 if lo_parts else 0.0)
    W2 = np.zeros((width, width))
    b2 = np.zeros(width)
    b2[0] = 2.0 ** -5
    for j in range(1, width):
        b2[j] = 0.25 + rng.choice([-1, 1]) * 2.0 ** -14
        W2[j, 0] = -8.0
        c1, c2 = rng.choice(np.arange(1, width), size=2, replace=False)
        W2[j, c1] = rng.choice([-2, -1, 1, 2])
        W2[j, c2] = rng.choice([-1, 1])
    W3 = np.zeros((3, width))
    b3 = rng.choice([-1, 1], size=3) * rng.integers(32, 64, size=3) / 128 + rng.choice([-1, 1], size=3) * 2.0 ** -14
    for c in range(3):
        for k in rng.choice(np.arange(width), size=4, replace=False):
            W3[c, k] = rng.choice([-4, -2, -1, 1, 2, 4])
    diff = None if direct else rng.integers(-16, 17, size=(n, 3)) / 16.0
    w = 2.0 ** -rng.integers(0, 5, size=n).astype(np.float64)
    return [(W1, b1), (W2, b2), (W3, b3)], x, diff, w


def exact_logits(layers, x, diff, split=False, check=True):
    """fp64 logits; split: the f16x3 products hi*hi + lo*hi + hi*lo of layer 1 (the lo*lo term dropped by design);
    check: assert that the hidden values are fp16-exact."""
    (W1, b1), (W2, b2), (W3, b3) = layers
    if split:
        xh, Wh = f16(x), f16(W1)
        xl, Wl = f16(x - xh), f16(W1 - Wh)
        a = xh @ Wh.T + xl @ Wh.T + xh @ Wl.T + b1
    else:
        a = x @ W1.T + b1
    h1 = np.maximum(a, 0)
    h2 = np.maximum(h1 @ W2.T + b2, 0)
    lg = h2 @ W3.T + b3
    if check and not split:
        assert np.array_equal(f16(h1), h1) and np.array_equal(f16(h2), h2), 'hidden values are not fp16-exact'
    return lg + (diff if diff is not None else 0.0)



@pytest.mark.parametrize('spec', MODELS, ids=MODEL_IDS)
def test_exact_operands_all_modes_bit_identical(cuda_device, spec):
    rng = np.random.default_rng(zlib.crc32(spec[0].encode()))
    name, kind, c, vpe, spe, width, direct, cid = spec
    dim0 = dim0_of(kind, c, vpe, spe, direct)
    layers, x, diff, w = exact_operands(dim0, width, direct, max(ROWS), rng)
    m = Model(spec, layers, cuda_device)
    assert np.array_equal(np.array(m.layers[0][1]), layers[0][1]), 'biases must survive fp32'
    for n in ROWS:
        lg = exact_logits(layers, x[:n], None if diff is None else diff[:n])
        want = w[:n, None] * sig(lg)
        rows = {}
        for mode in MODES:
            G = group_size(mode)
            owner = perm_owners(n, G, rng)
            st, racc, Gk = m.run(mode, x[:n], None if diff is None else diff[:n], w[:n], owner)
            if not m.supports(mode):
                assert st == -2, (mode, st)
                continue
            assert st == 0 and Gk == G, (mode, st, Gk)
            rows[mode] = per_row(racc, owner, G)
            assert unowned_zero(racc, owner, G), (n, mode, 'an owner without rows received colour')
            err = np.abs(rows[mode] - want)
            assert (err <= SIG_REL * want).all(), (n, mode, float((err / want).max() / SIG_REL))
        ref = rows['fp32']
        for mode, r in rows.items():
            assert np.array_equal(r, ref), (n, mode, int((r != ref).sum()), float(np.abs(r - ref).max()))


@pytest.mark.parametrize('spec', [s for s in MODELS if supports(s, 'f16x3')], ids=[s[0] for s in MODELS if supports(s, 'f16x3')])
def test_f16x3_keeps_the_lo_parts_exactly(cuda_device, spec):
    """f16x3 on operands with non-zero fp16 lo parts (exact_operands(lo_parts=True)): bit-exact against the fp64 sum of
    its three products, which differs from the hi-only sum of single-pass f16 in most rows."""
    rng = np.random.default_rng(7 + zlib.crc32(spec[0].encode()))
    name, kind, c, vpe, spe, width, direct, cid = spec
    dim0 = dim0_of(kind, c, vpe, spe, direct)
    layers, x, diff, w = exact_operands(dim0, width, direct, 300, rng, lo_parts=True)
    m = Model(spec, layers, cuda_device)
    lg = exact_logits(layers, x, diff, split=True)
    hi_only = exact_logits([(f16(layers[0][0]), layers[0][1])] + layers[1:], f16(x), diff, check=False)
    assert (np.abs(lg - hi_only).max(axis=1) >= 2.0 ** -22).mean() > 0.9, 'the lo parts must matter'
    owner = perm_owners(300, 32, rng)
    st, racc, G = m.run('f16x3', x, diff, w, owner)
    assert st == 0
    got = per_row(racc, owner, G)
    want = w[:, None] * sig(lg)
    assert (np.abs(got - want) <= SIG_REL * want).all(), float((np.abs(got - want) / want).max() / SIG_REL)


@pytest.mark.parametrize('spec', MODELS, ids=MODEL_IDS)
def test_wgmma_inputs_saturate_to_fp16_max(cuda_device, spec):
    """Inputs beyond the fp16 range enter the wgmma rows as +-65504 (h2_sat is cvt.rn.satfinite), never as inf."""
    rng = np.random.default_rng(11)
    name, kind, c, vpe, spe, width, direct, cid = spec
    dim0 = dim0_of(kind, c, vpe, spe, direct)
    layers, x, diff, w = exact_operands(dim0, width, direct, 200, rng)
    layers = [(W / 1024.0, b) if i == 0 else (W, b) for i, (W, b) in enumerate(layers)]
    m = Model(spec, layers, cuda_device)
    big = x.copy()
    sel = rng.random(big.shape) < 0.2
    big[sel] = rng.choice([65519.0, 65520.0, 7e4, 1e6, 3e38, -65520.0, -1e9], size=int(sel.sum()))
    owner = perm_owners(200, 128, rng)
    st, r_big, _ = m.run('ws', big, diff, w, owner)
    st2, r_clamp, _ = m.run('ws', np.clip(big, -65504.0, 65504.0), diff, w, owner)
    assert st == 0 and st2 == 0
    assert np.isfinite(r_big).all() and np.array_equal(r_big, r_clamp)


# ---------------------------------------------------------------------------------------------------------------------
# b / c. random operands, per-element bound
# ---------------------------------------------------------------------------------------------------------------------
def realistic_inputs(kind, c, vpe, spe, direct, n, rng):
    """k0 ~ N(0, 1), the view embedding of real unit directions, MPI position codes of points in [-1, 1]^3."""
    def emb(v, nf):
        f = 2.0 ** np.arange(nf)
        return np.concatenate([v, np.sin(v[:, :, None] * f).reshape(n, -1), np.cos(v[:, :, None] * f).reshape(n, -1)], 1)
    k0 = rng.standard_normal((n, c))
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    parts = [k0 if direct else k0[:, 3:]]
    if kind == 'cfgB':
        parts.append(emb(rng.uniform(-1, 1, (n, 3)), spe))
    parts.append(emb(d, vpe))
    x = np.concatenate(parts, 1).astype(np.float32).astype(np.float64)
    diff = None if direct else k0[:, :3].astype(np.float32).astype(np.float64)
    return x, diff


def random_layers(dim0, width, seed):
    torch.manual_seed(seed)
    ls = [torch.nn.Linear(dim0, width), torch.nn.Linear(width, width), torch.nn.Linear(width, 3)]
    return [(l.weight.detach().double().numpy(), l.bias.detach().double().numpy()) for l in ls]


def racc_check(mode, m, x, diff, w, owner, G, racc):
    """Per owner: |racc - sum w sigma(ref)| <= sum w (sigma'_max E + 3.5 * 2^-23 sigma_hi) + (n_o - 1) u sum w sigma_hi.
    Returns (largest error / bound, median logit bound)."""
    lg, E = logit_bound(mode, m, x, diff)
    zc = np.clip(0.0, lg - E, lg + E)
    dmax = sig(zc) * (1 - sig(zc))
    s_hi = sig(lg + E)
    row_ref = w[:, None] * sig(lg)
    row_b = w[:, None] * (dmax * E + 3.5 * 2.0 ** -23 * s_hi)
    row_hi = w[:, None] * s_hi
    ng = racc.shape[0]
    g = np.arange(x.shape[0]) // G
    ref, bnd, hi, cnt = (np.zeros((ng, G, 3)) for _ in range(4))
    np.add.at(ref, (g, owner), row_ref)
    np.add.at(bnd, (g, owner), row_b)
    np.add.at(hi, (g, owner), row_hi)
    np.add.at(cnt, (g, owner), 1.0)
    bnd += np.maximum(cnt - 1, 0) * U * hi
    err = np.abs(racc - ref)
    ok = (err <= bnd) & np.isfinite(racc)
    assert ok.all(), (mode, int((~ok).sum()), float((err / np.maximum(bnd, 1e-300)).max()))
    return float((err / np.maximum(bnd, 1e-300)).max()), float(np.median(E))


RATIOS = {}


@pytest.mark.parametrize('spec', MODELS, ids=MODEL_IDS)
def test_random_operands_within_bound(cuda_device, spec):
    """nn.Linear default initialisation, realistic inputs; every row its own owner (b), then many rows per owner (c)."""
    rng = np.random.default_rng(3)
    name, kind, c, vpe, spe, width, direct, cid = spec
    dim0 = dim0_of(kind, c, vpe, spe, direct)
    m = Model(spec, random_layers(dim0, width, seed=cid + 100 * width + dim0), cuda_device)
    x, diff = realistic_inputs(kind, c, vpe, spe, direct, 300, rng)
    w = np.maximum(rng.random(300), 1e-3).astype(np.float32).astype(np.float64)
    med = {}
    for mode in MODES:
        if not m.supports(mode):
            continue
        G = group_size(mode)
        for n in ROWS:
            xs, ds, ws = x[:n], None if diff is None else diff[:n], w[:n]
            for owner in (perm_owners(n, G, rng), rng.integers(0, 3, size=n).astype(np.int32)):
                st, racc, Gk = m.run(mode, xs, ds, ws, owner)
                assert st == 0 and Gk == G
                r, med[mode] = racc_check(mode, m, xs, ds, ws, owner, G, racc)
                RATIOS[mode] = max(RATIOS.get(mode, 0.0), r)
    if 'f16x3' in med:
        RATIOS['f16x3/f16 bound'] = max(RATIOS.get('f16x3/f16 bound', 0.0), med['f16x3'] / med['f16'])
    print(spec[0], 'largest error/bound so far', {k: f'{v:.3g}' for k, v in RATIOS.items()})


# ---------------------------------------------------------------------------------------------------------------------
# 3. per ray: every tensor-core mode against fp32 mode, with the per-sample inputs of the CPU oracle
# ---------------------------------------------------------------------------------------------------------------------
def check_per_ray_against_fp32(m, st, spec, rays, kw, runs, dev, label, act=None):
    """Renders `runs` ((mode, image_hw) pairs) and fp32 mode (in the first run's order) and bounds every run's colour per
    ray against fp32's.  The marchers march bit-identically in every mode, so per ray the colours of a tensor-core mode
    and of fp32 mode differ only through the MLP on the same samples.  The oracle's trace gives each shaded sample's
    weight and rgbnet inputs; per sample both logits lie within their bounds of the unquantised fp64 model
    (true_logit_bound, or mpi_act.act_logit_bound for a hidden activation `act`), so

        |rgb_mode - rgb_fp32| <= sum_i w_i [sigma'_max (L_mode,i + L_fp32,i) + 2 * SIG_REL * sigma_hi + 2 u sigma_hi]
                                 + 2 (n - 1) u sum_i w_i sigma_hi + 2 u |rgb|

    (the two sigmoids, the two products w * sigma, the two sums of n terms, the two background adds).  The GPU weight of a
    sample is taken as the oracle's times 1 + 1e-4, and the GPU inputs within FEAT_REL of the oracle's.  Every run's
    alphainv_last and ray_stats equal fp32's on every ray.  Rays whose in-box, occupied or shaded sample counts differ
    from the oracle's (a sample at a threshold) are left out of the bound; at most 1e-3 of the rays may be.
    Returns (n_c, bad): the oracle's shaded samples per ray and the rays left out."""
    from oracle import ops, pipeline
    import contextlib
    import mpi_act
    ro, rd, vd = rays
    stats, trace = {}, {}
    with mpi_act.oracle_act(act) if act else contextlib.nullcontext():
        ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, trace=trace, **kw)
    args = (ro.to(dev), rd.to(dev), vd.to(dev), kw)
    fp = m.render_rays(*args, image_hw=runs[0][1], mlp_mode='fp32', debug=True)
    outs = {(mode, hw): m.render_rays(*args, image_hw=hw, mlp_mode=mode, debug=True) for mode, hw in runs}
    torch.cuda.synchronize()
    fp = {n: t.cpu() for n, t in fp.items()}
    N = ro.shape[0]
    rid = trace['ray_id'].long()
    n_c = torch.bincount(rid, minlength=N)
    rs, ors = fp['ray_stats'].long(), ref['_ray_stats']
    bad = (rs[:, 1] != ors[:, 0]) | (rs[:, 2] != ors[:, 1]) | (rs[:, 3] != n_c)
    assert int(bad.sum()) <= max(1, int(1e-3 * N)), (label, int(bad.sum()))

    shp = shape_info(types.SimpleNamespace(), spec)
    shp.layers = [(w_.double().numpy(), b_.double().numpy()) for w_, b_ in st['rgbnet']]
    x = trace['rgb_feat'].double().numpy()
    diff = None if trace['diffuse'] is None else trace['diffuse'].double().numpy()
    w = trace['weights'].double().numpy()[:, None] * (1 + 1e-4)
    D0 = FEAT_REL * np.abs(x) + 2.0 ** -24
    if act:
        bound = lambda mode: mpi_act.act_logit_bound(mode, shp, x, diff, act, D0=D0, true=True)
    else:
        bound = lambda mode: true_logit_bound(mode, shp, x, diff, D0)
    l_f, E_f = bound('fp32')
    rid_np = rid.numpy()
    rgb_f = fp['rgb_marched'].double()
    keep = ~bad.numpy()
    ratios = {}
    for key, o in outs.items():
        o = {n: t.cpu() for n, t in o.items()}
        assert torch.equal(o['alphainv_last'], fp['alphainv_last']) and torch.equal(o['ray_stats'], fp['ray_stats']), (label, key)
        l_m, E_m = bound(key[0])
        assert np.allclose(l_m, l_f, rtol=0, atol=1e-12)
        Em = np.maximum(E_m, E_f)
        zc = np.clip(0.0, l_f - Em, l_f + Em)
        dmax = sig(zc) * (1 - sig(zc))
        s_hi = sig(l_f + Em)
        per = w * (dmax * (E_m + E_f) + (2 * SIG_REL + 2 * U) * s_hi)
        B = np.zeros((N, 3))
        H = np.zeros((N, 3))
        np.add.at(B, rid_np, per)
        np.add.at(H, rid_np, w * s_hi)
        B += 2 * np.maximum(n_c.numpy()[:, None] - 1, 0) * U * H + 2 * U * rgb_f.abs().numpy()
        d = (o['rgb_marched'].double() - rgb_f).abs().numpy()
        ok = d[keep] <= B[keep]
        assert ok.all(), (label, key, int((~ok).sum()), float((d[keep] / np.maximum(B[keep], 1e-300)).max()))
        ratios[key] = float((d[keep] / np.maximum(B[keep], 1e-300)).max())
    print(label, 'per-ray error/bound against fp32', {k: f'{v:.3g}' for k, v in ratios.items()})
    return n_c, bad


def _ray_spec(kind, skw, cid):
    return ('ray', kind, skw['k0_dim'], skw['viewbase_pe'], skw.get('spatial_pe', 0), skw['width'],
            int(skw.get('rgbnet_direct', True)), cid)


# the rgbnet shapes of make_state's default DirectVoxGO (configs/default.py fine stage) and DirectMPIGO (LLFF) scenes
WS_RING_SPECS = {'cfgA': _ray_spec('cfgA', dict(k0_dim=12, viewbase_pe=4, width=128), 1),
                 'cfgB': _ray_spec('cfgB', dict(k0_dim=9, viewbase_pe=0, spatial_pe=0, width=64), 6)}


def ws_both_orders(hw):
    """ws on image tiles (when the rays form an image) and in flat ray order."""
    return [('ws', hw), ('ws', None)] if hw else [('ws', None)]


@pytest.mark.parametrize('kind', ['cfgA', 'cfgB'])
@pytest.mark.parametrize('regime', ['fog', 'shell', 'blobs'])
def test_ws_against_fp32_per_ray(cuda_device, kind, regime):
    if regime == 'blobs':
        st = _blob_state(kind)
    else:
        st = make_state(kind, xy=48, depth=32, regime=regime) if kind == 'cfgB' else make_state(kind, res=48, regime=regime)
    hw = (40, 52)
    rays, kw = rays_for(st, *hw)
    m = model_from_state(st, cuda_device)
    n_c, _ = check_per_ray_against_fp32(m, st, WS_RING_SPECS[kind], rays, kw, ws_both_orders(hw), cuda_device, (kind, regime))
    assert int(n_c.sum()) > 1000


def test_ring_long_queues_next_to_empty_rays(cuda_device):
    """fast_color_thres 0 and thin fog: a few rays queue more than 384 samples (one group's queue spans several ring
    tiles) while their neighbours miss the volume."""
    st = make_state('cfgA', res=48, regime='fog')
    st['fast_color_thres'] = 0.0
    st['density'] = torch.full_like(st['density'], -9.0)
    (ro, rd, vd), kw = rays_for(st, 16, 16)
    kw['stepsize'] = 0.05                           # more than 1000 steps through the 48^3 grid
    far = torch.tensor([0.0, 0.0, 50.0]).expand(256, 3).clone()
    keep = torch.zeros(256, dtype=torch.bool)
    keep[[3, 77, 140, 141, 255]] = True
    ro = torch.where(keep[:, None], ro, far)
    m = model_from_state(st, cuda_device)
    n_c, bad = check_per_ray_against_fp32(m, st, WS_RING_SPECS['cfgA'], (ro, rd, vd), kw, ws_both_orders(None), cuda_device, 'long')
    assert not bad[keep].any()
    assert int(n_c.max()) > 384 and int((n_c == 0).sum()) >= 200, (int(n_c.max()), int((n_c == 0).sum()))


def test_ring_one_live_ray_per_tile(cuda_device):
    """Linear ray order with exactly one ray per 128-ray tile inside the volume: every MLP batch is partial."""
    st = make_state('cfgA', res=48, regime='fog')
    (ro, rd, vd), kw = rays_for(st, 32, 64)
    n = ro.shape[0]
    keep = torch.zeros(n, dtype=torch.bool)
    keep[torch.arange(37, n, 128)] = True
    ro = torch.where(keep[:, None], ro, torch.tensor([0.0, 0.0, 50.0]))
    m = model_from_state(st, cuda_device)
    n_c, bad = check_per_ray_against_fp32(m, st, WS_RING_SPECS['cfgA'], (ro, rd, vd), kw, ws_both_orders(None), cuda_device, 'sparse')
    assert int(keep.sum()) == 16 and not bad[keep].any()
    assert int((n_c > 0).sum()) == int(keep.sum()) and int(n_c.max()) > 0


def test_ring_many_tiles_per_cta(cuda_device):
    """A 320 x 128 frame: 320 tiles of 16 x 8 pixels, more than the 2 x 132 marcher groups of the persistent grid, so
    56 groups take a second tile and run their FULL / DONE mbarriers on across a tile boundary."""
    st = make_state('cfgA', res=48, regime='shell')
    hw = (128, 320)
    rays, kw = rays_for(st, *hw)
    m = model_from_state(st, cuda_device)
    n_c, _ = check_per_ray_against_fp32(m, st, WS_RING_SPECS['cfgA'], rays, kw, ws_both_orders(hw), cuda_device, 'many tiles')
    assert int(n_c.sum()) > 100000


def test_f16x3_without_shared_memory_room_is_unsupported(cuda_device):
    """k0 16 with 6 view frequencies at width 128 (configuration 5): k4_render_rays in f16x3 reports an unsupported
    configuration -- it used to fail in cudaFuncSetAttribute with a CUDA error -- while f16 renders."""
    from k4nerf import _lib
    st = make_state('cfgA', res=24, regime='fog', k0_dim=16, viewbase_pe=6, width=128)
    (ro, rd, vd), kw = rays_for(st, 8, 8)
    m = model_from_state(st, cuda_device)
    ro, rd, vd = ro.to(cuda_device), rd.to(cuda_device), vd.to(cuda_device)
    with pytest.raises(_lib.K4Error, match='unsupported configuration'):
        m.render_rays(ro, rd, vd, kw, mlp_mode='f16x3')
    out = m.render_rays(ro, rd, vd, kw, mlp_mode='f16')
    torch.cuda.synchronize()
    assert torch.isfinite(out['rgb_marched']).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3b. per ray: every tensor-core mode against fp32 mode on every WS_SHAPES model
# ---------------------------------------------------------------------------------------------------------------------
RAY_SHAPES = [('cfgA', dict(k0_dim=12, viewbase_pe=4, width=128), 1),       # configs/default.py fine stage
              ('cfgB', dict(k0_dim=9, viewbase_pe=0, spatial_pe=0, width=64), 6)] + WS_SHAPES


@pytest.mark.parametrize('kind,skw,cfg_id', RAY_SHAPES,
                         ids=[f'{k}-{"-".join(f"{a}{b}" for a, b in v.items())}' for k, v, _ in RAY_SHAPES])
def test_tensor_core_modes_against_fp32_per_ray(cuda_device, kind, skw, cfg_id):
    """check_per_ray_against_fp32 for every tensor-core mode the shape has a build for, on image tiles; the others
    report an unsupported configuration."""
    from k4nerf import _lib
    dev = cuda_device
    if kind == 'cfgB':
        st = make_state(kind, xy=40, depth=24, regime='fog', **skw)
        hw = (24, 32)
    else:
        st = make_state(kind, res=40, regime='fog', **skw)
        hw = (32, 40)
    rays, kw = rays_for(st, *hw, **({'radius': 0.6} if kind == 'cfgC' else {}))
    m = model_from_state(st, dev)
    spec = _ray_spec(kind, skw, cfg_id)
    runs = []
    for mode in ('f16', 'f16x3', 'ws'):
        if supports(spec, mode):
            runs.append((mode, hw))
        else:
            with pytest.raises(_lib.K4Error, match='unsupported configuration'):
                m.render_rays(*[t.to(dev) for t in rays], kw, image_hw=hw, mlp_mode=mode)
    n_c, _ = check_per_ray_against_fp32(m, st, spec, rays, kw, runs, dev, (kind, skw))
    assert int(n_c.sum()) > 1000
