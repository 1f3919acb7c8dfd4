"""CPU: the compositions of march_batches.py hit their per-tile row targets in both ray orders, the host replay of the
marchers' batch counts gives an empty 'ws' batch in exactly the tiles that end on a 128-row boundary while a ray still
marches, and on these scenes every shaded sample's colour w * sigma is far above every per-ray error bound the GPU test
holds the marchers to, so a lost, doubled or misattributed MLP row cannot pass it."""
import numpy as np
import pytest
import torch

import march_batches as mb
from march_bounds import sig, true_logit_bound, types_ns
from test_gpu_march_geometry import check_tc_against_fp32, check_values, fp64_reference, tc_bounds

MARGIN = 25.0       # smallest per-sample w * sigma against the largest per-ray bound


def frame(kind, order):
    ws = mb.ws_tiles(kind)
    wp = mb.warp_tiles(kind)
    return ws, wp, mb.layout(mb.target_tiles(kind), kind, order)


@pytest.mark.parametrize('order', ['linear', 'image'])
@pytest.mark.parametrize('cfg', [1, 6, 10], ids=['dvgo', 'dmpigo', 'dcvgo'])
def test_compositions_hit_their_targets(cfg, order):
    kind = mb.kind_of(cfg)
    ws, wp, (ro, rd, vd, hw, pos) = frame(kind, order)
    st = mb.scene(cfg)
    ref, trace, stats = mb.oracle(st, ro, rd, vd)
    # every occupied in-box sample is shaded, with alpha near ALPHA, and no ray comes near the early-out
    assert stats['S_c'] == stats['S_d'] > 0
    a = trace['composited']['alpha'].double()
    assert float(a.min()) > 3e-3 and float(a.max()) < 5e-3
    assert float(ref['alphainv_last'].min()) > 0.8
    rep = mb.replay(trace, mb.n_steps_of(st, ref, ro.shape[0]), hw)
    n_t, empty = rep['n_t'], rep['empty']
    tid = mb.tile_ids(ro.shape[0], hw, 16, 8)
    mid = mb.tile_ids(ro.shape[0], hw, 8, 4)
    for t, (name, n, want_empty, _) in enumerate(ws):
        k = tid[pos[t, 0, 0]]
        assert (tid[pos[t]] == k).all()
        assert n_t[k] == n, (name, n_t[k])
        assert bool(empty[k]) == want_empty, name
    # the empty batch comes in exactly the tiles on a 128-row boundary whose rays still march
    assert int(empty.sum()) == sum(1 for x in ws if x[2]) >= 4
    if kind != 'dcvgo':
        assert sum(1 for x in ws if x[1] % 128 == 0 and x[1] > 0 and not x[2]) >= 4
    for t, (name, ns, _) in enumerate(wp):
        for w in range(4):
            k = mid[pos[len(ws) + t, w, 0]]
            assert (mid[pos[len(ws) + t, w]] == k).all()
            assert rep['n_w'][k] == ns[w], (name, w, rep['n_w'][k])
    # the overflow tile: 50 rows on its first shading step, then 128 per step -- each appended with 50 pending
    t = [x[0] for x in ws].index('overflow')
    sel = np.isin(trace['ray_id'].numpy(), pos[t].ravel())
    per_step = np.bincount(trace['step_id'].numpy()[sel])
    per_step = per_step[per_step > 0]
    assert per_step[0] == 50 and (per_step[1:-1] == 128).all() and per_step[-1] == 78 and len(per_step) > 20
    pend = np.cumsum(per_step)[:-1] % 128
    assert ((per_step[1:] == 128) & (pend == 50)).sum() == len(per_step) - 2
    assert rep['ws_lo'] == sum(-(-int(n) // 128) for n in n_t)
    assert rep['ws'] == rep['ws_lo'] + sum(1 for x in ws if x[2])
    assert rep['ws_hi'] == rep['ws_lo'] + sum(1 for x in ws if x[1] % 128 == 0 and x[1] > 0)


@pytest.mark.parametrize('cfg', sorted(mb.CFGS))
def test_bounds_cannot_hide_a_lost_or_doubled_row(cfg):
    """The per-ray bounds of the GPU test (fp32 against the fp64 recomposition, every tensor-core mode against fp32) are
    below 1/25 of the smallest per-sample colour on these scenes, and a recomposition that drops or repeats one sample
    fails both comparisons."""
    kind = mb.kind_of(cfg)
    _, _, (ro, rd, vd, hw, _) = frame(kind, 'linear')
    st = mb.scene(cfg)
    ref, trace, _ = mb.oracle(st, ro, rd, vd)
    N = ro.shape[0]
    ref64 = fp64_reference(st, trace, N, mb.KWS[kind], set())
    modes = [m for m in mb.modes_of(st) if m != 'fp32']
    bounds = tc_bounds(st, trace, ref64, ref64['rgb'], modes)
    shp = types_ns(st)
    x = trace['rgb_feat'].double().numpy()
    diff = None if trace['diffuse'] is None else trace['diffuse'].double().numpy()
    lg, _ = true_logit_bound('fp32', shp, x, diff)
    wsig = trace['weights'].double().numpy()[:, None] * sig(lg)
    worst = max([float(ref64['B'].max())] + [float(b.max()) for b in bounds.values()])
    print(f'config {cfg}: smallest w sigma {wsig.min():.4g}, largest per-ray bound {worst:.4g} '
          f'({", ".join(f"{m}: {float(b.max()):.3g}" for m, b in bounds.items())}, fp32 vs fp64: {float(ref64["B"].max()):.3g})')
    assert wsig.min() >= MARGIN * worst
    # a render equal to the recomposition passes; one with a sample dropped or repeated fails
    rid = trace['ray_id'].long().numpy()
    fake = dict(rgb_marched=torch.tensor(ref64['rgb'], dtype=torch.float32), depth=torch.tensor(ref64['depth'], dtype=torch.float32),
                alphainv_last=torch.tensor(ref64['T'], dtype=torch.float32))
    check_values(fake, ref64, 'exact', {})
    for j in (0, len(rid) // 2, len(rid) - 1):
        for sgn in (-1.0, 1.0):
            bad = dict(fake, rgb_marched=fake['rgb_marched'].clone())
            bad['rgb_marched'][rid[j]] += torch.tensor(sgn * wsig[j], dtype=torch.float32)
            with pytest.raises(AssertionError):
                check_values(bad, ref64, 'one sample off', {})
            for m in modes:
                with pytest.raises(AssertionError):
                    check_tc_against_fp32(fake, {(False, m, None): bad}, st, trace, ref64, set(), 'one sample off', {})
