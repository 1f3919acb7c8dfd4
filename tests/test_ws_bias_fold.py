"""Layer 1's bias inside K on the warp-specialised marcher's configurations (csrc/k4_ws_cfgs.h, k4_ws_bias_col).

Where a configuration's A row has two spare columns below its layer-1 K (the first even column at or past its input
count, and the next), the rows carry fp16 1.0 there and W1 the bias hi / lo, so the bias products ride in layer 1's last
k16 step instead of one more MMA against a tile of ones.  The CPU test checks every configuration's compiled row layout
against the config list; the GPU tests run the same zero-padded model on an unfolded configuration and on a folded one
(K4_WS_CONFIG) and compare them per owner: bit for bit on exact operands, within the reordering of the fp32 sums on random
ones, and per ray through the marcher, whose ring rows carry the ones.
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from march_bounds import SIG_REL, WS_CFGS, dim0_of, sig


def expected_layout(kind, c, vpe, spe, direct):
    """(dim0, kpad, bias column or -1, row store writes it) of a configuration, from its shape."""
    ns = (c if direct else c - 3) + (3 + 6 * spe if kind == 'cfgB' else 0)
    dim0 = (ns + 1) // 2 * 2 + 3 + 6 * vpe
    kpad = (dim0 + 15) // 16 * 16
    col = (dim0 + 1) // 2 * 2
    if col + 1 >= kpad:
        return dim0, kpad, -1, 0
    return dim0, kpad, col, int((col // 2) % 4 != 0)


@pytest.mark.parametrize('cfg', WS_CFGS, ids=[f'cfg{c[0]}' for c in WS_CFGS])
def test_row_layout_matches_the_config_list(cfg):
    from k4nerf import _lib
    cid, kind, c, vpe, spe, w, direct = cfg
    out = (C.c_int32 * 4)()
    assert _lib.lib.k4_testing_ws_row_layout(cid, out) == 0
    dim0, kpad, col, stored = expected_layout(kind, c, vpe, spe, direct)
    assert tuple(out) == (dim0, kpad, col, stored), (cid, tuple(out))
    assert dim0 >= dim0_of(kind, c, vpe, spe, direct)          # the model of the config's own shape fits its row
    if col >= 0:
        assert col >= dim0 and col % 2 == 0 and col + 1 < kpad
    else:
        assert kpad - dim0 < 2 + dim0 % 2                       # no even pair left below kpad


def test_fold_decision_of_the_shipped_configs():
    """Every configuration with view frequencies folds; the four with kpad 16 (15 inputs) keep the ones-tile MMA."""
    from k4nerf import _lib
    out = (C.c_int32 * 4)()
    cols = {}
    for cfg in WS_CFGS:
        assert _lib.lib.k4_testing_ws_row_layout(cfg[0], out) == 0
        cols[cfg[0]] = out[2]
    assert cols == {0: -1, 2: -1, 6: -1, 9: -1, 1: 40, 3: 40, 4: 40, 10: 40, 5: 56, 11: 56, 7: 44, 8: 74}


def test_unknown_config_is_rejected():
    from k4nerf import _lib
    out = (C.c_int32 * 4)(7, 7, 7, 7)
    assert _lib.lib.k4_testing_ws_row_layout(99, out) == -1 and tuple(out) == (0, 0, 0, 0)
    assert _lib.lib.k4_testing_ws_row_layout(0, None) == -1


# (name, kind, C, vpe, spe, width, direct): a model whose first covering configuration keeps the ones-tile MMA, and a
# folded configuration that also covers it: 3 and 1 set the ones once per ring, the row store of 7 and 8 writes them
PAIRS = [
    (('dvgo-w64', 'cfgA', 12, 0, 0, 64, 1), 2, 3),
    (('dvgo-w128', 'cfgA', 12, 0, 0, 128, 1), 0, 1),
    (('mpi-w64', 'cfgB', 9, 0, 0, 64, 1), 6, 7),
    (('mpi-w64-pe', 'cfgB', 9, 0, 0, 64, 1), 6, 8),
]
PAIR_IDS = [f'{p[0][0]}-cfg{p[1]}-cfg{p[2]}' for p in PAIRS]


def _pair_models(shape, plain, folded, layers, dev, monkeypatch):
    from k4nerf import _lib
    from test_gpu_march_mlp import Model
    ms = []
    for cid in (plain, folded):
        monkeypatch.setenv('K4_WS_CONFIG', str(cid))
        m = Model((*shape, cid), layers, dev)
        assert _lib.lib.k4_scene_ws_config(m.m._get_scene().ptr) == cid
        monkeypatch.delenv('K4_WS_CONFIG')
        ms.append(m)
    return ms


@pytest.mark.gpu
@pytest.mark.parametrize('shape,plain,folded', PAIRS, ids=PAIR_IDS)
def test_folded_equals_unfolded_on_exact_operands(cuda_device, monkeypatch, shape, plain, folded):
    """Exact operands (test_gpu_march_mlp.exact_operands: layer-1 biases with non-zero fp16 lo parts, every sum exact in
    any order): the two configurations agree bit for bit per owner, and with the fp64 colours."""
    from test_gpu_march_mlp import ROWS, exact_logits, exact_operands, per_row, perm_owners, unowned_zero
    name, kind, c, vpe, spe, width, direct = shape
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    dim0 = dim0_of(kind, c, vpe, spe, direct)
    layers, x, diff, w = exact_operands(dim0, width, direct, max(ROWS), rng)
    assert (np.float16(layers[0][1][1:]).astype(np.float64) != layers[0][1][1:]).all(), 'the lo parts must be non-zero'
    ma, mb = _pair_models(shape, plain, folded, layers, cuda_device, monkeypatch)
    for n in ROWS:
        want = w[:n, None] * sig(exact_logits(layers, x[:n], None))
        owner = perm_owners(n, 128, rng)
        rows = []
        for m in (ma, mb):
            st, racc, G = m.run('ws', x[:n], None, w[:n], owner)
            assert st == 0 and G == 128
            assert unowned_zero(racc, owner, G), (n, m.cid)
            rows.append(per_row(racc, owner, G))
        assert np.array_equal(rows[0], rows[1]), (n, int((rows[0] != rows[1]).sum()), float(np.abs(rows[0] - rows[1]).max()))
        assert (np.abs(rows[1] - want) <= SIG_REL * want).all(), n


@pytest.mark.gpu
@pytest.mark.parametrize('shape,plain,folded', PAIRS, ids=PAIR_IDS)
def test_folded_equals_unfolded_on_random_operands(cuda_device, monkeypatch, shape, plain, folded):
    """Random weights and inputs: the products are the same in both configurations, only the order of the fp32 sums in
    layer 1 differs, so the colours agree to a few ulp of the logits; 1e-4 relative leaves room for a hidden value that
    the reordering moves across an fp16 rounding boundary, and is far below what a lost or doubled bias costs."""
    from helpers import make_state
    name, kind, c, vpe, spe, width, direct = shape
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 1)
    st = make_state(kind, res=8, regime='fog', k0_dim=c, viewbase_pe=vpe, width=width) if kind == 'cfgA' else \
        make_state(kind, xy=8, depth=8, regime='fog', k0_dim=c, viewbase_pe=vpe, spatial_pe=spe, width=width)
    layers = [(W.double().numpy(), b.double().numpy() + rng.normal(0, 0.3, b.shape[0])) for W, b in st['rgbnet']]
    ma, mb = _pair_models(shape, plain, folded, layers, cuda_device, monkeypatch)
    n = 1000
    x = rng.normal(0, 1, (n, dim0_of(kind, c, vpe, spe, direct)))
    w = rng.uniform(0.1, 1.0, n)
    owner = rng.integers(0, 128, n).astype(np.int32)
    ra = ma.run('ws', x, None, w, owner)[1]
    rb = mb.run('ws', x, None, w, owner)[1]
    assert np.isfinite(ra).all() and np.isfinite(rb).all()
    d = np.abs(ra - rb)
    assert (d <= 1e-4 * np.abs(ra) + 1e-6).all(), float(d.max())


@pytest.mark.gpu
@pytest.mark.parametrize('shape,plain,folded', PAIRS, ids=PAIR_IDS)
def test_folded_equals_unfolded_per_ray(cuda_device, monkeypatch, shape, plain, folded):
    """The marcher on both configurations: the same samples (geometry is untouched by the rgbnet) and per-ray colours
    within the reordering of layer 1's sums."""
    from helpers import make_state, model_from_state, rays_for
    from k4nerf import _lib
    name, kind, c, vpe, spe, width, direct = shape
    st = make_state(kind, res=48, regime='fog', k0_dim=c, viewbase_pe=vpe, width=width) if kind == 'cfgA' else \
        make_state(kind, xy=40, depth=24, regime='fog', k0_dim=c, viewbase_pe=vpe, spatial_pe=spe, width=width)
    (ro, rd, vd), kw = rays_for(st, 40, 56)
    ro, rd, vd = ro.to(cuda_device), rd.to(cuda_device), vd.to(cuda_device)
    outs = []
    for cid in (plain, folded):
        monkeypatch.setenv('K4_WS_CONFIG', str(cid))
        m = model_from_state(st, cuda_device)
        assert _lib.lib.k4_scene_ws_config(m._get_scene().ptr) == cid
        monkeypatch.delenv('K4_WS_CONFIG')
        outs.append(m.render_rays(ro, rd, vd, kw, image_hw=(40, 56), mlp_mode='ws', debug=True))
    torch.cuda.synchronize()
    a, b = outs
    assert torch.equal(a['alphainv_last'], b['alphainv_last'])
    assert torch.equal(a['ray_stats'], b['ray_stats'])
    assert int(a['ray_stats'][:, 3].sum()) > 1000, 'the scene must shade samples'
    d = (a['rgb_marched'] - b['rgb_marched']).abs()
    assert float(d.max()) <= 1e-4, float(d.max())
