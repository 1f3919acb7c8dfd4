"""Helpers of the DirectMPIGO activation tests (test_mpi_act.py on the CPU, test_gpu_mpi_act.py on the GPU).

The reference's act_type (lib/dmpigo.py:89-95) puts one activation module after every hidden nn.Linear of the rgbnet:
'relu', 'gauss' (GaussianActivation(a=0.05), lib/act.py) or 'lkrelu' (nn.LeakyReLU()).  This file holds
  * the torch restatement of that Sequential (mlp_act) and a context that runs oracle/pipeline.py with it (oracle_act);
  * scenes whose rgbnet exercises the activation (scale_for_act): with nn.Linear's default initialisation the
    pre-activations are about +-0.5, and at a = 0.05 the Gaussian is ~0 almost everywhere, so every colour would be
    sigmoid(b3) and every comparison would pass trivially;
  * the fp64 error model of the kernels with the activation (act_logit_bound), the model of march_bounds.py with its
    ReLU step replaced: a pre-activation error e becomes at most e * max|g'| over [z - e, z + e] (the mean value
    theorem), plus the error of evaluating g in fp32 and, in the fp16 modes, the rounding of the activated value.
"""
import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import pipeline
from march_bounds import GAMMA_TC, U, f16

A_GAUSS = 0.05                                  # GaussianActivation(a=0.05), lib/dmpigo.py:93
LK_SLOPE = float(np.float32(0.01))             # nn.LeakyReLU(): negval 0.01 applied in fp32 (ATen leaky_relu)
ACTS = ('gauss', 'lkrelu')
K4_ACT = {'relu': 0, 'gauss': 1, 'lkrelu': 2}


# ---------------------------------------------------------------------------------------------------------------------
# torch restatement (the oracle side)
# ---------------------------------------------------------------------------------------------------------------------
def torch_act(x, act, a=A_GAUSS):
    """The reference module's forward on x (any dtype); ``a`` as GaussianActivation holds it, a one-element fp32
    parameter, so 2*a**2 is rounded in fp32 as in the reference."""
    if act == 'relu':
        return F.relu(x)
    if act == 'gauss':
        at = torch.full((1,), float(a), dtype=torch.float32, device=x.device).to(x.dtype)
        return torch.exp(-x ** 2 / (2 * at ** 2))
    if act == 'lkrelu':
        return F.leaky_relu(x)
    raise ValueError(act)


def mlp_act(layers, x, act, a=A_GAUSS):
    """nn.Sequential(Linear, act, [Linear, act], ..., Linear) of lib/dmpigo.py:100-105 on (W, b) pairs."""
    for i, (w, b) in enumerate(layers):
        x = F.linear(x, w, b)
        if i + 1 < len(layers):
            x = torch_act(x, act, a)
    return x


@contextlib.contextmanager
def oracle_act(act, a=A_GAUSS):
    """oracle/pipeline.py's forward with the rgbnet's hidden activation `act` (its own mlp is the ReLU Sequential)."""
    orig = pipeline.mlp
    pipeline.mlp = lambda layers, x: mlp_act(layers, x, act, a)
    try:
        yield
    finally:
        pipeline.mlp = orig


# ---------------------------------------------------------------------------------------------------------------------
# scenes that exercise the activation
# ---------------------------------------------------------------------------------------------------------------------
def pre_activations(layers, x, act, a=A_GAUSS):
    """fp64 pre-activations [z1, z2] of the two hidden layers (layers: (W, b) numpy float64)."""
    zs, h = [], x
    for W, b in layers[:-1]:
        z = h @ W.T + b
        zs.append(z)
        h = np_act(z, act, a)
    return zs


def scale_for_act(layers, x, act, a=A_GAUSS, target=2.0):
    """For gauss: scale W_l and b_l of the two hidden layers, in turn, so that the RMS of their pre-activations over
    the inputs x is `target` * a (the Gaussian then spans (1e-3, 0.999) for most units).  Other activations: unchanged.
    Returns new float32-representable (W, b) pairs as float64 numpy arrays."""
    out = [(np.asarray(W, np.float64).copy(), np.asarray(b, np.float64).copy()) for W, b in layers]
    if act != 'gauss':
        return out
    h = x
    for i in range(len(out) - 1):
        W, b = out[i]
        z = h @ W.T + b
        s = target * a / max(float(np.sqrt(np.mean(z ** 2))), 1e-30)
        W = (W * s).astype(np.float32).astype(np.float64)
        b = (b * s).astype(np.float32).astype(np.float64)
        out[i] = (W, b)
        h = np_act(h @ W.T + b, act, a)
    return out


def coverage(layers, x, act, a=A_GAUSS):
    """(fraction of the hidden outputs in (1e-3, 0.999), fraction of negative pre-activations), both hidden layers."""
    zs = pre_activations(layers, x, act, a)
    z = np.concatenate([q.ravel() for q in zs])
    g = np_act(z, act, a)
    return float(((g > 1e-3) & (g < 0.999)).mean()), float((z < 0).mean())


def assert_exercised(layers, x, act, a=A_GAUSS):
    cov, neg = coverage(layers, x, act, a)
    if act == 'gauss':
        assert cov >= 0.25, ('the Gaussian is saturated on this scene', cov)
    if act == 'lkrelu':
        assert neg >= 0.25, ('too few negative pre-activations for LeakyReLU', neg)
    return cov, neg


def scale_state_rgbnet(st, act, n=4096, seed=0, a=A_GAUSS):
    """scale_for_act on an oracle MPI state, with inputs drawn like the marcher's: k0 at random voxels of the grid, the
    position code of random points in [-1, 1]^3, the view embedding of random unit directions.  Returns those inputs."""
    x = sample_inputs(st, n, seed)
    layers = [(W.double().numpy(), b.double().numpy()) for W, b in st['rgbnet']]
    st['rgbnet'] = [(torch.tensor(W, dtype=torch.float32), torch.tensor(b, dtype=torch.float32))
                    for W, b in scale_for_act(layers, x, act, a)]
    return x


def sample_inputs(st, n, seed):
    rng = np.random.default_rng(seed)
    k0 = st['k0'][0].reshape(st['k0'].shape[1], -1).double().numpy()
    x_k0 = k0[:, rng.integers(0, k0.shape[1], n)].T

    def emb(v, nf):
        f = 2.0 ** np.arange(nf)
        return np.concatenate([v, np.sin(v[:, :, None] * f).reshape(n, -1), np.cos(v[:, :, None] * f).reshape(n, -1)], 1)
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x = np.concatenate([x_k0, emb(rng.uniform(-1, 1, (n, 3)), len(st['posfreq'])), emb(d, len(st['viewfreq']))], 1)
    return x.astype(np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# the product model
# ---------------------------------------------------------------------------------------------------------------------
def mpi_model(st, act, device=None, a=A_GAUSS):
    """k4nerf.DirectMPIGO with act_type=`act` and the oracle state's tensors (tests/helpers.model_from_state builds
    the relu model only)."""
    import k4nerf
    from k4nerf._scene import linear_layers
    kw = dict(xyz_min=st['xyz_min'].tolist(), xyz_max=st['xyz_max'].tolist(), num_voxels=st['_num_voxels'],
              mpi_depth=st['mpi_depth'], fast_color_thres=st['fast_color_thres'], rgbnet_dim=st['rgbnet_dim'],
              mask_cache_world_size=list(st['mask_cache']['mask'].shape), act_type=act, mode_type='mlp',
              rgbnet_depth=len(st['rgbnet']), rgbnet_width=st['rgbnet'][0][0].shape[0],
              viewbase_pe=len(st['viewfreq']), spatial_pe=len(st['posfreq']))
    m = k4nerf.DirectMPIGO(**kw)
    sd = m.state_dict()
    sd['density.grid'] = st['density'].clone()
    sd['k0.grid'] = st['k0'].clone()
    sd['mask_cache.mask'] = st['mask_cache']['mask'].clone()
    names = {id(mod): n for n, mod in m.rgbnet.named_modules()}
    for lin, (w, b) in zip(linear_layers(m.rgbnet), st['rgbnet']):
        sd['rgbnet.' + names[id(lin)] + '.weight'] = w.clone()
        sd['rgbnet.' + names[id(lin)] + '.bias'] = b.clone()
    if act == 'gauss':
        for k in sd:
            if k.startswith('rgbnet.') and k.endswith('.a'):
                sd[k] = torch.full((1,), float(a))
    m.load_state_dict(sd)
    if device is not None:
        m = m.to(device)
    return m


# ---------------------------------------------------------------------------------------------------------------------
# fp64 error model
# ---------------------------------------------------------------------------------------------------------------------
def np_act(z, act, a=A_GAUSS):
    if act == 'relu':
        return np.maximum(z, 0)
    if act == 'gauss':
        return np.exp(-z ** 2 / (2 * a * a))
    return np.where(z > 0, z, LK_SLOPE * z)


def max_dact(lo, hi, act, a=A_GAUSS):
    """max |g'| over [lo, hi] (elementwise)."""
    if act != 'gauss':
        return np.ones_like(lo)
    h = lambda u: u / (a * a) * np.exp(-u * u / (2 * a * a))           # |g'| at |x| = u, rising to u = a, then falling
    umin = np.where((lo <= 0) & (hi >= 0), 0.0, np.minimum(np.abs(lo), np.abs(hi)))
    umax = np.maximum(np.abs(lo), np.abs(hi))
    return np.where((umin <= a) & (umax >= a), h(a), np.maximum(h(umin), h(umax)))


# Evaluating g in fp32, on the exact fp32 input:
#  fp32 mode, gauss: x*x (u), 2*(a*a) rounded on the host (2u against 2 a^2 of the fp32 a), the division (u), expf (2 ulp):
#    the exponent t = -x^2/(2a^2) is off by 4u |t|, so the value by 4u |t| e^-|t| <= 4u/e, plus 2 ulp <= 4u g.
#  tc modes, gauss: x*x and *c (2u), c rounded from double (u): 3u |t'| on t' = log2 g, i.e. 3u ln2 |t'| 2^-|t'| <= 3u/e;
#    ex2.approx.ftz: 2^-22 relative (PTX ISA: maximum relative error 2^-22 over the full range) and 2^-126 absolute
#    (flush to zero).
#  lkrelu: one product 0.01 * x (u relative); relu exact.
def act_eval_err(g_hi, act, tc):
    if act == 'gauss':
        return (2.0 ** -22 * g_hi + 3 * U / math.e + 2.0 ** -126) if tc else (4 * U * g_hi + 4 * U / math.e + 2.0 ** -149)
    if act == 'lkrelu':
        return U * g_hi
    return 0.0 * g_hi


def _act_step(z, E, act, a, tc):
    """(activated fp64 value of the model, bound on the kernel's activated value's distance from it, before any fp16
    rounding of the kernel)."""
    g = np_act(z, act, a)
    g_hi = np.maximum(np.abs(np_act(z - E, act, a)), np.abs(np_act(z + E, act, a)))
    if act == 'gauss':
        g_hi = np.where((z - E <= 0) & (z + E >= 0), 1.0, g_hi)
    return g, E * max_dact(z - E, z + E, act, a) + act_eval_err(g_hi, act, tc)


def act_logit_bound(mode, m, x, diff, act, a=A_GAUSS, D0=None, true=False):
    """march_bounds.logit_bound (true=False: f16 / ws held to the fp16-quantised model) or true_logit_bound (true=True:
    every mode held to the unquantised fp64 model) with the hidden activation `act`.  Returns (logits [n, 3], bound)."""
    wg = mode == 'ws'
    tc = mode != 'fp32'
    layers = m.layers
    if mode in ('f16', 'ws') and not true:
        h = f16(np.clip(x, -65504, 65504))
        D = np.zeros_like(h)
        ks = [m.kpad_cfg, m.w_cfg, m.w_cfg] if wg else [m.kpad_mma, m.width, m.width]
        for i, (W, b) in enumerate(layers):
            Wq = f16(W)
            bias = f16(b) + f16(b - f16(b)) if wg else b
            n_instr = ks[i] // 16 + (1 if wg else 0)
            z = h @ Wq.T + bias
            S = (np.abs(h) + D) @ np.abs(Wq).T + np.abs(bias)
            E = D @ np.abs(Wq).T + n_instr * GAMMA_TC * S
            if i < 2:
                g, Eg = _act_step(z, E, act, a, tc)
                h = f16(g)
                # both sides round to fp16: |f16(y) - y| <= 2^-11 |y| + 2^-25
                D = Eg + 2 * (2.0 ** -11 * (np.abs(g) + Eg) + 2.0 ** -25)
        lg = z
    elif mode == 'f16x3':
        h, D = x, (np.zeros_like(x) if D0 is None else D0)
        ks = [m.kpad_mma, m.width, m.width]
        for i, (W, b) in enumerate(layers):
            av = np.abs(h) + D
            ev, lv = 2.0 ** -22 * av + 2.0 ** -25, 2.0 ** -11 * av + 2.0 ** -24
            aw = np.abs(W)
            ew, lw = 2.0 ** -22 * aw + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -24
            split = lv @ lw.T + av @ ew.T + ev @ aw.T + ev @ ew.T
            z = h @ W.T + b
            S = av @ aw.T + av @ lw.T + lv @ aw.T + np.abs(b)
            E = D @ aw.T + split + 3 * (ks[i] // 16) * GAMMA_TC * S
            if i < 2:
                h, D = _act_step(z, E, act, a, tc)
        lg = z
    elif mode == 'fp32':
        h, D = x, (np.zeros_like(x) if D0 is None else D0)
        for i, (W, b) in enumerate(layers):
            z = h @ W.T + b
            S = (np.abs(h) + D) @ np.abs(W).T + np.abs(b)
            E = D @ np.abs(W).T + W.shape[1] * U * S
            if i < 2:
                h, D = _act_step(z, E, act, a, tc)
        lg = z
    else:
        ks = [m.kpad_cfg, m.w_cfg, m.w_cfg] if wg else [m.kpad_mma, m.width, m.width]
        h, D = x, (np.zeros_like(x) if D0 is None else D0)
        for i, (W, b) in enumerate(layers):
            av, aw = np.abs(h) + D, np.abs(W)
            ea, ew = 2.0 ** -11 * av + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -25
            eb = 2.0 ** -22 * np.abs(b) + 2.0 ** -25 if wg else 0.0
            z = h @ W.T + b
            S = (av + ea) @ (aw + ew).T + np.abs(b)
            E = D @ aw.T + ea @ aw.T + av @ ew.T + ea @ ew.T + eb + (ks[i] // 16 + (1 if wg else 0)) * GAMMA_TC * S
            if i < 2:
                h, D = _act_step(z, E, act, a, tc)
        lg = z
    if diff is not None:
        E = E + U * (np.abs(lg) + E + np.abs(diff))
        lg = lg + diff
    return lg, E
