"""GPU: how the marchers cut their shaded samples into MLP batches, on scenes whose per-tile row counts are chosen
(march_batches.py): tiles that end before, on and after every 128-row ('ws') and 32-row (f16 / f16x3) boundary,
a tile ending on a boundary while a ray still marches ('ws' sends an empty batch that only carries `last`), a step that
appends 128 rows with 50 pending, and a ring that wraps many times -- one tile per marcher group, and a frame of 24
times as many tiles, so the groups carry their FULL / DONE phases from tile to tile.  Configurations 1 and 2
(DirectVoxGO; the fine-stage shape and the ones-tile build), 6 and 7 (DirectMPIGO; the LLFF shape and the build that
stores the bias word with each row) and 10 (DirectContractedVoxGO).

Per render (every mode the shape has, image and linear order, empty-space skipping on and off):
  * counters[3] against the host replay of march_batches.replay: equal without skipping, within its range with it;
  * ray_stats, alphainv_last and depth identical in every mode, ray_stats equal to the oracle's; a ray with no shaded
    sample exactly T * bg;
  * fp32 colour within the fp64 recomposition's bound, every tensor-core mode within its per-ray bound of fp32 mode
    (test_gpu_march_geometry.py), bounds that are below 1/25 of any one sample's colour (test_march_batches.py).
"""
import pytest
import torch

import march_batches as mb
from test_gpu_march_geometry import (check_geometry, check_modes_agree, check_tc_against_fp32, check_values,
                                     fp64_reference, models, render_all)

pytestmark = pytest.mark.gpu
RATIOS = {}


def run(st, ms, rays, label):
    ro, rd, vd, hw = rays[:4]
    N = ro.shape[0]
    kw = mb.KWS[st['kind']]
    bg = float(kw['bg'])
    ref, trace, stats = mb.oracle(st, ro, rd, vd)
    outs = render_all(ms, ro, rd, vd, kw, hw, mb.modes_of(st))
    base = check_modes_agree(outs, hw, bg, label)
    for key, o in outs.items():
        none = o['ray_stats'][:, 3] == 0
        assert torch.equal(o['rgb_marched'][none], (o['alphainv_last'][none] * bg)[:, None].expand(-1, 3)), (label, key)
    assert not check_geometry(base, ref, trace, st, N, label)
    assert torch.equal(base['ray_stats'][:, 3].long(), torch.bincount(trace['ray_id'].long(), minlength=N))
    ref64 = fp64_reference(st, trace, N, kw, set())
    ratios = {}
    check_values(base, ref64, label, ratios)
    check_tc_against_fp32(base, {k: o for k, o in outs.items() if k[1] != 'fp32'}, st, trace, ref64, set(), label, ratios)
    # batch counts ('skip' is a no-op for DirectContractedVoxGO, which has no empty-space skipping)
    n_steps = mb.n_steps_of(st, ref, N)
    reps = {}
    lines = []
    for (skip, mode, order), o in sorted(outs.items(), key=lambda kv: (kv[0][0], kv[0][1], kv[0][2] is None)):
        if mode == 'fp32':
            continue
        if order not in reps:
            reps[order] = mb.replay(trace, n_steps, order)
        rep = reps[order]
        got = int(o['counters'][3])
        if mode in ('f16', 'f16x3'):
            lo = hi = rep['f16']
        elif skip and st['kind'] != 'dcvgo':
            lo, hi = rep['ws_lo'], rep['ws_hi']
        else:
            lo = hi = rep['ws']
        want = f'{lo}' if lo == hi else f'{lo}..{hi}'
        lines.append(f'{mode}/{"image" if order else "linear"}/{"skip" if skip else "noskip"} {want}/{got}')
        assert lo <= got <= hi, (label, skip, mode, order, 'expected', want, 'got', got)
    for k, v in ratios.items():
        RATIOS[k] = max(RATIOS.get(k, 0.0), v)
    print(f'[{label}] rays {N}  rows {int(base["counters"][2])}  batches expected/got: {", ".join(lines)}  '
          f'largest error/bound {{{", ".join(f"{k}: {v:.3g}" for k, v in ratios.items())}}}  '
          f'all cases so far {{{", ".join(f"{k}: {v:.3g}" for k, v in RATIOS.items())}}}')


CFGS = sorted(mb.CFGS)


@pytest.mark.parametrize('cfg', CFGS)
def test_batch_counts_at_their_boundaries(cuda_device, monkeypatch, cfg):
    """One tile per marcher group: every target tile laid out in linear order and, as 16 x 8 blocks, in image order."""
    st = mb.scene(cfg)
    kind = mb.kind_of(cfg)
    ms = models(st, cuda_device, monkeypatch)
    for order in ('linear', 'image'):
        run(st, ms, mb.layout(mb.target_tiles(kind), kind, order), f'config {cfg} targets {order}')


@pytest.mark.parametrize('cfg', CFGS)
def test_batch_counts_across_tiles(cuda_device, monkeypatch, cfg):
    """The target tiles 24 times over (in image order 24 blocks wide) on 2 x 132 marcher groups: every group takes
    several tiles and runs its FULL / DONE phases on across them, among them tiles after an empty last batch."""
    st = mb.scene(cfg)
    kind = mb.kind_of(cfg)
    ms = models(st, cuda_device, monkeypatch)
    tiles = mb.target_tiles(kind) * 24
    assert len(tiles) > 2 * 132
    run(st, ms, mb.layout(tiles, kind, 'image', tx=24), f'config {cfg} frame')
