"""Error bounds of the marchers' colour MLP against float64 references, shared by the GPU tests of the rgbnet
(test_gpu_march_mlp.py) and of the marchers' geometry and compositing (test_gpu_march_geometry.py).

The error model is documented in test_gpu_march_mlp.py's module docstring (u = 2^-24, the unit roundoff of fp32).
"""
import numpy as np

U = 2.0 ** -24
GAMMA_TC = 17 * 2.0 ** -23          # one MMA instruction, relative to S (module docstring)


# csrc/k4_ws_cfgs.h, K4_WS_CFG_LIST: id, kind, C, viewbase_pe, spatial_pe, width, rgbnet_direct
WS_CFGS = [(2, 'cfgA', 12, 0, 0, 64, 1), (0, 'cfgA', 12, 0, 0, 128, 1), (3, 'cfgA', 12, 4, 0, 64, 1), (1, 'cfgA', 12, 4, 0, 128, 1),
           (4, 'cfgA', 15, 4, 0, 128, 0), (5, 'cfgA', 16, 6, 0, 128, 1), (6, 'cfgB', 9, 0, 0, 64, 1), (7, 'cfgB', 12, 4, 0, 128, 1),
           (8, 'cfgB', 12, 4, 5, 128, 1), (9, 'cfgC', 12, 0, 0, 128, 1), (10, 'cfgC', 12, 4, 0, 128, 1), (11, 'cfgC', 16, 6, 0, 128, 1)]


def dim0_of(kind, c, vpe, spe, direct):
    k0 = c if direct else c - 3
    return k0 + (3 + 6 * spe if kind == 'cfgB' else 0) + 3 + 6 * vpe


def supports(spec, mode):
    """The modes a model shape has a build for.  mma.sync (f16 / f16x3): widths 64 / 128 and up to 64 inputs; f16x3
    keeps two weight parts and two rows per ring slot in shared memory, which do not fit a block (227 KB) at width 128
    with more than 48 inputs.  fp32 and ws: every shape here."""
    name, kind, c, vpe, spe, w, direct, cid = spec
    kpad = (dim0_of(kind, c, vpe, spe, direct) + 15) // 16 * 16
    if mode in ('f16', 'f16x3'):
        return kpad <= 64 and w in (64, 128) and not (mode == 'f16x3' and w == 128 and kpad > 48)
    return True


def f16(a):
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


def sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def shape_info(obj, spec):
    """The K extents the kernels run: kpad_mma (mma.sync layer 1), kpad_cfg / w_cfg (the wgmma configuration)."""
    name, kind, c, vpe, spe, w, direct, cid = spec
    obj.spec, obj.width = spec, w
    obj.dim0 = dim0_of(kind, c, vpe, spe, direct)
    obj.kpad_mma = (obj.dim0 + 15) // 16 * 16
    _, ckind, cc, cvpe, cspe, cw, cd = next(x for x in WS_CFGS if x[0] == cid)
    ns = (cc if cd else cc - 3) + (3 + 6 * cspe if ckind == 'cfgB' else 0)
    obj.kpad_cfg = ((ns + 1) // 2 * 2 + 3 + 6 * cvpe + 15) // 16 * 16
    obj.w_cfg = cw
    return obj


# sigmoid_ref against the exact sigmoid of an exact logit: expf within 2 ulp, the add and the division within 1/2 ulp each,
# 3 * 2^-23 relative to first order; 2^-40 covers the second-order terms.  w = 2^-e makes w * sigma exact.
SIG_REL = 3 * 2.0 ** -23 + 2.0 ** -40


def logit_bound(mode, m, x, diff, D0=None):
    """(reference logits [n, 3], bound on |kernel logit - reference| [n, 3]) of one mode (module docstring).  The
    f16 / wgmma reference is quantised as the kernel is; fp32 and f16x3 are held to the unquantised model.  D0 (fp32 and
    f16x3 only) bounds the difference between the kernel's inputs and x."""
    layers = m.layers
    wg = mode == 'ws'
    if mode in ('f16', 'ws'):
        a = f16(np.clip(x, -65504, 65504))
        D = np.zeros_like(a)
        ks = [m.kpad_cfg, m.w_cfg, m.w_cfg] if wg else [m.kpad_mma, m.width, m.width]
        for i, (W, b) in enumerate(layers):
            Wq = f16(W)
            bias = f16(b) + f16(b - f16(b)) if wg else b
            n_instr = ks[i] // 16 + (1 if wg else 0)
            z = a @ Wq.T + bias
            S = (np.abs(a) + D) @ np.abs(Wq).T + np.abs(bias)
            E = D @ np.abs(Wq).T + n_instr * GAMMA_TC * S
            if i < 2:
                a = f16(np.maximum(z, 0))
                D = f16(np.maximum(z + E, 0)) - f16(np.maximum(z - E, 0))
        lg = z
    elif mode == 'f16x3':
        a, D = x, (np.zeros_like(x) if D0 is None else D0)
        ks = [m.kpad_mma, m.width, m.width]
        for i, (W, b) in enumerate(layers):
            av = np.abs(a) + D
            ev, lv = 2.0 ** -22 * av + 2.0 ** -25, 2.0 ** -11 * av + 2.0 ** -24
            aw = np.abs(W)
            ew, lw = 2.0 ** -22 * aw + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -24
            split = lv @ lw.T + av @ ew.T + ev @ aw.T + ev @ ew.T
            z = a @ W.T + b
            S = av @ aw.T + av @ lw.T + lv @ aw.T + np.abs(b)
            E = D @ aw.T + split + 3 * (ks[i] // 16) * GAMMA_TC * S
            if i < 2:
                a, D = np.maximum(z, 0), E
        lg = z
    else:
        a, D = x, (np.zeros_like(x) if D0 is None else D0)
        for i, (W, b) in enumerate(layers):
            z = a @ W.T + b
            S = (np.abs(a) + D) @ np.abs(W).T + np.abs(b)
            E = D @ np.abs(W).T + W.shape[1] * U * S
            if i < 2:
                a, D = np.maximum(z, 0), E
        lg = z
    if diff is not None:
        E = E + U * (np.abs(lg) + E + np.abs(diff))
        lg = lg + diff
    return lg, E


def true_logit_bound(mode, m, x, diff, D0=None):
    """(logits of the unquantised fp64 model, bound on |kernel logit - those| [n, 3]) for any mode; D0 bounds the
    difference between the kernel's inputs and x.  f16 / wgmma round inputs, weights and hidden values to fp16:
    |v - fp16(v)| <= 2^-11 |v| + 2^-25; the wgmma bias hi + lo misses at most 2^-22 |b| + 2^-25."""
    if mode in ('fp32', 'f16x3'):
        return logit_bound(mode, m, x, diff, D0)
    wg = mode == 'ws'
    ks = [m.kpad_cfg, m.w_cfg, m.w_cfg] if wg else [m.kpad_mma, m.width, m.width]
    a, D = x, (np.zeros_like(x) if D0 is None else D0)
    for i, (W, b) in enumerate(m.layers):
        av, aw = np.abs(a) + D, np.abs(W)
        ea, ew = 2.0 ** -11 * av + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -25
        eb = 2.0 ** -22 * np.abs(b) + 2.0 ** -25 if wg else 0.0
        z = a @ W.T + b
        S = (av + ea) @ (aw + ew).T + np.abs(b)
        E = D @ aw.T + ea @ aw.T + av @ ew.T + ea @ ew.T + eb + (ks[i] // 16 + (1 if wg else 0)) * GAMMA_TC * S
        if i < 2:
            a, D = np.maximum(z, 0), E
    lg = z
    if diff is not None:
        E = E + U * (np.abs(lg) + E + np.abs(diff))
        lg = lg + diff
    return lg, E


def types_ns(st):
    """The rgbnet shape of an oracle scene as shape_info describes it, with its layers in float64.  The configuration is
    the one of WS_CFGS with the scene's exact shape."""
    import types
    kind = {'dvgo': 'cfgA', 'dmpigo': 'cfgB', 'dcvgo': 'cfgC'}[st['kind']]
    key = (kind, st['k0_dim'], len(st['viewfreq']), len(st.get('posfreq', [])), st['rgbnet'][0][0].shape[0],
           int(st.get('rgbnet_direct', True)))
    cid = next(x[0] for x in WS_CFGS if x[1:] == key)
    o = shape_info(types.SimpleNamespace(), ('geo', *key, cid))
    o.layers = [(a.double().numpy(), b.double().numpy()) for a, b in st['rgbnet']]
    return o


FEAT_REL = 2.0 ** -16      # GPU sample inputs against the oracle's (trilinear k0, sin / cos): far below this, relative
