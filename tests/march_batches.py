"""Scenes whose per-tile shaded sample counts are chosen, and a host replay of the marchers' MLP batch counts
(test_march_batches.py on the CPU, test_gpu_march_batches.py on the GPU).

Scenes, one per model kind, all with fast_color_thres = 0 and a density that gives every sample alpha = ALPHA, so every
occupied in-box sample is shaded and T stays far above the 1e-3 early-out.  The occupancy mask is a slab and the rays are
parallel to one axis (exact geometry); h is the distance between samples:
  DirectVoxGO      box [-1, 1]^3, 32^3, occupied for x < 0; rays along x, stepsize 0.5 (h = 1 / 32.5), near 0.1.
  DirectMPIGO      box [-1, 1]^3, 32 x 32 x 32 planes, occupied for z > 0 (the act_shift grid is cancelled in the
                   density); rays along z over 63 samples spaced h = 1 / 32.5.
  DirectContracted foreground [-1, 1]^3 (unit frame = world frame), 32^3 over [-1.2, 1.2]^3, occupied for
  VoxGO            -0.93 < x < 0 and |y|, |z| < 0.93 (no contracted sample is occupied); rays along x, h = 2 / 54.
Ray families (a spec is (family, count)):
  END k     shades k samples and ends on the last.  DirectVoxGO: a -x ray from inside the slab, k steps.  DirectMPIGO: a
            +z ray whose last k samples are in the slab, so it shades on the step it ends on (every MPI ray has all 63).
  MARCH k   shades its first k samples, then keeps marching: DirectVoxGO 32 in-box empty steps, DirectMPIGO and
            DirectContractedVoxGO to the end of their fixed sample lists (at least 30 steps).
  ENTER e   e samples before the slab, then crosses it: 33 (DirectVoxGO), 32 (DirectMPIGO), 26 (DirectContractedVoxGO).
  PARK      a ray away from the box: nothing shaded (one step in DirectVoxGO, all of them in the other kinds).
DirectContractedVoxGO has no END family: its rays march all samples of the fixed list, whose last ones are contracted
points that the cumulative-distance rule keeps or drops, so no ray can be made to shade on its last step; its tiles that
end on a 128-row boundary all carry the empty batch.

A ray tile is four warps of 32 rays.  Laid out in linear order, tile t is rays [128 t, 128 t + 128) and its warp w
rays [128 t + 32 w, ..); laid out in image order (16 x 8 pixel blocks), the tile is block t and its warp w the 8 x 4 block
the 'ws' marcher gives warp w -- which is also the mma.sync marchers' warp tile.  So one composition pins the
rows of every 'ws' tile and of every mma.sync warp tile in both orders.

Batch counts (counters[3]) with K4_NO_SKIP=1, derived from k4_march_ws.cu / k4_march_mma.cuh:
  * 'ws': a batch whenever 128 rows are pending at a rendezvous, and one for a partial remainder: sum ceil(n_t / 128);
    plus an empty batch carrying only WgCtl::last for a tile whose rows end on a 128-row boundary while one of its rays
    still marches: the batch of the last 128 rows went out without `last` (tile_open).
  * f16 / f16x3: each warp flushes every 32 rows and once for a remainder: sum over warp tiles of ceil(n_w / 32).
The warps of a 'ws' group do not march in lockstep: between rendezvous each takes up to TC_ROUND steps and stops early
once 128 rows are pending, so one warp may run ahead of another, by more steps over a long tile.  Whether a ray is live
when the last full batch goes out therefore depends on which warp appends the tile's last row.  The compositions make
that not matter:
  * in a tile meant to end with `last`, every warp with rays in the box shades on its own last step, so the tile's last
    row is appended only after every warp has ended;
  * in a tile meant to send the empty batch, every warp has a ray that still marches at least 30 steps after the tile's
    last shaded step (DirectVoxGO: one MARCH ray per warp; the other kinds: every ray), so the warp that appends the last
    row is itself still live when it stops at the next pending check.
With skipping on, a marching ray may jump over its empty steps before the last full batch goes out, so 'ws' lies between
sum ceil(n_t / 128) and that plus the number of tiles with n_t a positive multiple of 128.
"""
import math

import numpy as np
import torch

from oracle import pipeline, scenes
from march_bounds import supports, types_ns

BOX = ([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0])
RES = 32
ALPHA = 4e-3
DELTA = 0.0011                  # offset of every sample from the slab's faces and the box's faces, in world units
MPI_N = 63                      # samples per DirectMPIGO ray: (mpi_depth - 1) / stepsize + 1
KWS = {'dvgo': dict(scenes.RENDER_KW_DVGO, near=0.1, bg=0.37),
       'dmpigo': dict(scenes.RENDER_KW_MPI, stepsize=0.5, bg=0.37),
       'dcvgo': dict(scenes.RENDER_KW_DCVGO, bg=0.37)}
# configuration id (csrc/k4_ws_cfgs.h) -> (kind, rgbnet shape):
#   1  DirectVoxGO, the fine stage of configs/default.py
#   2  DirectVoxGO, 'ws' with the ones-tile MMA: its 15 inputs fill layer 1's 16 columns, no padding column for the bias
#   6  DirectMPIGO, the LLFF shape
#   7  DirectMPIGO, 'ws' writing the bias word from the row store (BIAS_STORED)
#  10  DirectContractedVoxGO
CFGS = {1: ('dvgo', dict(rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4)),
        2: ('dvgo', dict(rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=64, viewbase_pe=0)),
        6: ('dmpigo', dict(rgbnet_dim=9, rgbnet_depth=3, rgbnet_width=64, viewbase_pe=0, spatial_pe=0)),
        7: ('dmpigo', dict(rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4, spatial_pe=0)),
        10: ('dcvgo', dict(rgbnet_dim=12, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4))}


def num_voxels(extent):
    """num_voxels for which a cubic box of the given extent comes out RES voxels wide (lib/dvgo.py:152-158)."""
    vs = extent / (RES + 0.5)
    return int(round(extent ** 3 / vs ** 3))


def _density_for(alpha, interval):
    """The pre-activation x with 1 - (1 + e^x)^-interval = alpha."""
    return math.log(math.expm1(-math.log1p(-alpha) / interval))


def scene(cfg):
    kind, shape = CFGS[cfg]
    if kind == 'dvgo':
        nv = num_voxels(2.0)
        st = pipeline.dvgo_state(*BOX, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=0.0,
                                 rgbnet_direct=True, **shape)
        st.update(_num_voxels=nv, _num_voxels_base=nv, _alpha_init=1e-2)
        scenes.fill_grids(st, 'fog')
    elif kind == 'dmpigo':
        st = pipeline.dmpigo_state(*BOX, num_voxels=RES ** 3, mpi_depth=RES, fast_color_thres=0.0, **shape)
        st['_num_voxels'] = RES ** 3
        scenes.fill_grids(st, 'fog')
    else:
        nv = num_voxels(2.4)
        st = pipeline.dcvgo_state(*BOX, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=0.0,
                                  **shape)
        st['kind'] = 'dvgo'
        scenes.fill_grids(st, 'fog')
        st['kind'] = 'dcvgo'
        st.update(_num_voxels=nv, _num_voxels_base=nv, _alpha_init=1e-2, _fg_min=BOX[0], _fg_max=BOX[1])
    assert tuple(st['density'].shape[2:]) == (RES,) * 3
    scenes.fill_rgbnet(st)
    # sigma near 1: a sample's colour w * sigma is about w, while the colour error of a tensor-core mode scales with
    # sigma' = sigma (1 - sigma)
    w3, b3 = st['rgbnet'][-1]
    st['rgbnet'][-1] = (w3, b3 + 6.0)
    kw = KWS[kind]
    if kind == 'dmpigo':
        # density + act_shift(z) = x on every plane, and so (both trilinear in z) at every sample
        x = _density_for(ALPHA, float(kw['stepsize']) * float(st['voxel_size_ratio']))
        st['density'] = (x - st['act_shift_grid']).expand(1, 1, RES, RES, RES).contiguous()
    else:
        x = _density_for(ALPHA, float(kw['stepsize']) * float(st['voxel_size_ratio']))
        st['density'] = torch.full_like(st['density'], x - float(st['act_shift']))
    mask = torch.zeros((RES,) * 3, dtype=torch.bool)
    if kind == 'dvgo':
        mask[:RES // 2] = True                   # mask voxel i <= 15 <=> x < 0 (scale 15.5, shift 15.5, roundf)
    elif kind == 'dmpigo':
        mask[:, :, RES // 2:] = True             # k >= 16 <=> z > 0
    else:
        mask[4:16, 4:28, 4:28] = True            # scale 31 / 2.4: x in [-0.929, 0), y and z in [-0.929, 0.929)
    st['mask_cache'] = pipeline.mask_grid_state(mask, st['xyz_min'], st['xyz_max'])
    return st


def kind_of(cfg):
    return CFGS[cfg][0]


def modes_of(st):
    shp = types_ns(st)
    return tuple(m for m in ('fp32', 'f16', 'f16x3', 'ws') if m == 'fp32' or supports(shp.spec, m))


def spacing(kind):
    if kind == 'dvgo':
        nv = num_voxels(2.0)
        st = pipeline.dvgo_state(*BOX, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=0.0)
        return float(np.float32(KWS['dvgo']['stepsize']) * np.float32(float(st['voxel_size'])))
    if kind == 'dmpigo':
        return 1.0 / 32.5
    n_inner = int(2 / 2.4 * RES / KWS['dcvgo']['stepsize']) + 1     # lib/dcvgo.py:240
    return 2.0 / n_inner


DCVGO_XLO = (3.5 - 15.5) / (31 / 2.4)            # the slab's lower x face in the mask (voxel 4 starts there)


def ray(spec, kind, h, rng):
    """(origin, direction) of one ray of a spec (module docstring)."""
    y, z = rng.uniform(-0.8, 0.8, 2)
    fam = spec[0]
    if fam == 'park':
        return (0.0, 0.0, 50.0), (0.0, 0.0, 1.0)
    k = spec[1]
    if kind == 'dvgo':
        if fam == 'end':
            start, d = -1.0 + (k - 0.5) * h + DELTA, -1.0
        elif fam == 'march':
            start, d = -(k - 0.5) * h + DELTA, 1.0
        else:
            start, d = (k - 0.5) * h + DELTA, -1.0
        return (start - d * KWS['dvgo']['near'], y, z), (d, 0.0, 0.0)
    if kind == 'dmpigo':
        L = (MPI_N - 1) * h                     # sample i at o + d i / (MPI_N - 1): h apart
        if fam == 'end':
            return (y, z, (k - 0.5) * h + DELTA - L), (0.0, 0.0, L)
        if fam == 'march':
            return (y, z, (k - 0.5) * h + DELTA), (0.0, 0.0, -L)
        return (y, z, -(k - 0.5) * h + DELTA), (0.0, 0.0, L)
    # DirectContractedVoxGO: sample i at t = (i + 1/2) h from the origin
    assert fam != 'end'
    if fam == 'march':
        return (-k * h + DELTA, y, z), (1.0, 0.0, 0.0)
    return (DCVGO_XLO + DELTA - (k + 0.5) * h, y, z), (1.0, 0.0, 0.0)


def split(n, size, rng, fam='end'):
    """size rays of family fam whose shaded counts add up to n (n // size or one more each; 0: parked), shuffled."""
    q, r = divmod(n, size)
    specs = [(fam, q + 1)] * r + ([(fam, q)] if q else [('park',)]) * (size - r)
    return [specs[i] for i in rng.permutation(size)]


def tile_of(specs):
    return [specs[32 * w:32 * w + 32] for w in range(4)]


def marching(specs, kind, n, rng):
    """A tile of n rows whose rays keep marching after its last row: DirectVoxGO turns one END ray per warp into a
    MARCH ray of the same count, the other kinds take MARCH rays throughout."""
    if kind != 'dvgo':
        return split(n, 128, rng, 'march')
    specs = list(specs)
    for w in range(4):
        j = next((32 * w + l for l in range(32) if specs[32 * w + l][0] == 'end'), None)
        if j is not None:
            specs[j] = ('march', specs[j][1])
    return specs


def ws_tiles(kind, seed=0):
    """[(name, n_t, empty last batch expected, tile)] for the 'ws' targets."""
    rng = np.random.default_rng(seed)
    base = 'end' if kind != 'dcvgo' else 'march'
    out = []
    for n in (0, 1, 127, 128, 129, 255, 256, 257, 383, 384, 385, 1024, 1100):
        specs = split(n, 128, rng, base)
        out.append((f'{n}', n, base == 'march' and n % 128 == 0 and n > 0, tile_of(specs)))
        if kind != 'dcvgo' and (n % 128 == 0 and n > 0 or n in (127, 385)):
            # the same number of rows with rays that still march when the tile's last row is appended: on a 128-row
            # boundary the last full batch goes without `last` and an empty one follows
            out.append((f'{n}-marching', n, n % 128 == 0, tile_of(marching(specs, kind, n, rng))))
    # overflow: 50 rays enter the slab on the first step, 78 on the next; while all 128 cross it every step appends 128
    # rows with 50 pending, so each one spills into the ring tile after the one filling, and the ring wraps many times
    specs = [('enter', 0)] * 50 + [('enter', 1)] * 78
    specs = [specs[i] for i in rng.permutation(128)]
    per_ray = {'dvgo': 33, 'dmpigo': 32, 'dcvgo': 26}[kind]
    out.append(('overflow', 128 * per_ray, kind != 'dvgo', tile_of(specs)))
    return out


WARP_TARGETS = (0, 1, 31, 32, 33, 63, 64, 65)


def warp_tiles(kind, seed=1):
    """[(name, (n_w of the four warps), tile)] for the mma.sync targets, two tiles of four warp targets."""
    rng = np.random.default_rng(seed)
    fam = 'end' if kind != 'dcvgo' else 'march'
    out = []
    for t in range(2):
        ns = WARP_TARGETS[4 * t:4 * t + 4]
        out.append((f'warps{ns}', ns, [split(n, 32, rng, fam) for n in ns]))
    return out


def target_tiles(kind):
    return [t[3] for t in ws_tiles(kind)] + [t[2] for t in warp_tiles(kind)]


def layout(tiles, kind, order, tx=None, seed=2):
    """Rays of the ray tiles (each four warps of 32 specs) laid out in 'linear' order or in 'image' order (tx tiles per
    row of 16 x 8 blocks).  Returns (ro, rd, vd, hw, pos) with hw None for linear order and pos[t, w, l] the index of
    lane l of warp w of tile t."""
    T = len(tiles)
    rng = np.random.default_rng(seed)
    h = spacing(kind)
    if order == 'linear':
        idx = lambda t, w, l: 128 * t + 32 * w + l
        N, hw = 128 * T, None
    else:
        tx = tx or T
        assert T % tx == 0
        H, W = 8 * (T // tx), 16 * tx
        idx = lambda t, w, l: ((t // tx) * 8 + (w >> 1) * 4 + (l >> 3)) * W + (t % tx) * 16 + (w & 1) * 8 + (l & 7)
        N, hw = H * W, (H, W)
    o = np.zeros((N, 3))
    d = np.zeros((N, 3))
    pos = np.zeros((T, 4, 32), np.int64)
    for t, tile in enumerate(tiles):
        for w in range(4):
            for l in range(32):
                pos[t, w, l] = idx(t, w, l)
                o[pos[t, w, l]], d[pos[t, w, l]] = ray(tile[w][l], kind, h, rng)
    ro = torch.tensor(o, dtype=torch.float32)
    rd = torch.tensor(d, dtype=torch.float32)
    return ro, rd, rd / rd.norm(dim=-1, keepdim=True), hw, pos


# ---------------------------------------------------------------------------------------------------------------------
# host replay of counters[3]
# ---------------------------------------------------------------------------------------------------------------------
def tile_ids(N, hw, bw, bh):
    """Per ray, the tile of bw x bh pixels (image order) or of bw * bh consecutive rays (linear order) it belongs to."""
    r = np.arange(N)
    if hw is None:
        return r // (bw * bh)
    H, W = hw
    return (r // W // bh) * ((W + bw - 1) // bw) + (r % W) // bw


def n_steps_of(st, ref, N):
    """Every ray's step count: DirectVoxGO's own, the fixed sample count of the other kinds."""
    if st['kind'] == 'dvgo':
        return ref['_N_steps'].long()
    n = MPI_N if st['kind'] == 'dmpigo' else int(ref['n_max'])
    return torch.full((N,), n, dtype=torch.long)


def replay(trace, n_steps, hw):
    """Per-tile rows and expected batch counts from the oracle's trace (module docstring).  n_steps: every ray's step
    count (n_steps_of).  Returns dict(n_t, empty, n_w, ws, ws_lo, ws_hi, f16) with n_t / empty per 'ws' tile and n_w
    per warp tile."""
    N = n_steps.shape[0]
    rid = trace['ray_id'].long().numpy()
    step = trace['step_id'].long().numpy()
    ns = n_steps.long().numpy()
    wt = tile_ids(N, hw, 16, 8)
    n_tiles = int(wt.max()) + 1
    n_t = np.bincount(wt[rid], minlength=n_tiles)
    last = np.full(n_tiles, -1)
    np.maximum.at(last, wt[rid], step)
    # a ray still active after its tile's last row: steps left beyond that row's step
    still = np.zeros(n_tiles, bool)
    np.logical_or.at(still, wt, ns - 1 > last[wt])
    empty = (n_t > 0) & (n_t % 128 == 0) & still
    mt = tile_ids(N, hw, 8, 4)
    n_w = np.bincount(mt[rid], minlength=int(mt.max()) + 1)
    full = int(sum(-(-int(n) // 128) for n in n_t))
    return dict(n_t=n_t, empty=empty, n_w=n_w, ws=full + int(empty.sum()),
                ws_lo=full, ws_hi=full + int(((n_t > 0) & (n_t % 128 == 0)).sum()),
                f16=int(sum(-(-int(n) // 32) for n in n_w)))


def oracle(st, ro, rd, vd):
    from oracle import ops
    trace, stats = {}, {}
    ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, trace=trace, **KWS[st['kind']])
    return ref, trace, stats
