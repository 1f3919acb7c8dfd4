"""Multi-GPU rendering of one frame: row-band sharding + one NCCL all-gather (SURVEY.md section 8e).

The reference has no multi-GPU path (its only NCCL code is vendored and unreachable, SURVEY.md
section 2.3), so this is new: rays are independent and the scene is read-only, hence every rank
holds a full replica of the scene (217 MB for 160^3 / 12 ch), marches its share of the image rows
with the same fused kernel -- 8-row blocks (the kernel's tile height) dealt round-robin over the
ranks, so that every rank gets the same mix of long and short rays -- and the shares are exchanged
with ONE ``all_gather_into_tensor`` of a packed ``[rgb(3) | depth | alphainv]`` buffer over
NVLink/NVSwitch.  No reduction crosses
GPUs, so results are bit-identical to the single-GPU render of the same rows.

Works with any ``torch.distributed`` backend (``nccl`` on GPUs; ``gloo`` in the CPU tests, where a
stand-in render function is injected because the kernel itself needs a GPU).
"""
import ctypes as C
import os

import torch
import torch.distributed as dist


ROW_BLOCK = 8      # height of the marcher's warpgroup tile (16x8 pixels): the unit of row interleaving


def cyclic_rows(H, rank, world_size, block=ROW_BLOCK):
    """Row indices of `rank` under block-cyclic sharding: 8-row blocks b with b % world == rank.
    Contiguous bands give the middle ranks the long rays (load imbalance = max over ranks); cyclic
    blocks give every rank the same mix.  Within a block the rows stay adjacent, so the kernel's
    16x8 pixel tiles keep their spatial locality."""
    nblk = (H + block - 1) // block
    rows = [torch.arange(b * block, min((b + 1) * block, H)) for b in range(rank, nblk, world_size)]
    return torch.cat(rows) if rows else torch.zeros(0, dtype=torch.long)


def cyclic_pad_rows(H, world_size, block=ROW_BLOCK):
    nblk = (H + block - 1) // block
    return ((nblk + world_size - 1) // world_size) * block


def unpack_frame_cyclic(gathered, H, W, world_size, block=ROW_BLOCK, out=None):
    """[world, 5 * n_pad] (block-cyclic bands) -> dict of full-frame tensors in image order.
    Image block b sits at local block b // world of rank b % world, so image order is the (local block,
    rank) transpose of the gathered buffer: one strided copy per quantity, no index kernels.
    ``out``: a ``[5 * world * n_pad]`` float buffer the three copies land in (the returned tensors are views
    of it, valid until it is written again); without it every call allocates the frame anew."""
    rows_pad = cyclic_pad_rows(H, world_size, block)
    n_pad = rows_pad * W
    nlb = rows_pad // block
    g = gathered.view(world_size, 5 * n_pad)
    if out is None:
        out = torch.empty(5 * world_size * n_pad, device=gathered.device, dtype=gathered.dtype)
    n_full = world_size * n_pad

    def image_order(x, c, dst):     # x: [world, rows_pad * W * c] -> dst: [nlb, world, block * W * c]
        dst.view(nlb, world_size, block * W * c).copy_(x.reshape(world_size, nlb, block * W * c).transpose(0, 1))
        return dst[:H * W * c]
    rgb = image_order(g[:, :3 * n_pad], 3, out[:3 * n_full]).view(H * W, 3)
    depth = image_order(g[:, 3 * n_pad:4 * n_pad], 1, out[3 * n_full:4 * n_full])
    ainv = image_order(g[:, 4 * n_pad:5 * n_pad], 1, out[4 * n_full:5 * n_full])
    return {'rgb_marched': rgb, 'depth': depth, 'alphainv_last': ainv}


def packed_band_views(buf, n_band_rays, n_pad_rays):
    """Views of a ``[5 * n_pad]`` packed band buffer (layout of :func:`pack_band`) that the marcher can write
    into directly (``render_rays(out=...)``): no pack copies.  The caller zero-fills the pad once at allocation."""
    return {'rgb_marched': buf[0:3 * n_band_rays].view(n_band_rays, 3),
            'depth': buf[3 * n_pad_rays:3 * n_pad_rays + n_band_rays],
            'alphainv_last': buf[4 * n_pad_rays:4 * n_pad_rays + n_band_rays]}


def band_rows(H, world_size):
    """Rows per band: every rank gets the same (padded) number of rows so that one
    fixed-size all-gather suffices."""
    return (H + world_size - 1) // world_size


def band_range(H, rank, world_size):
    rows = band_rows(H, world_size)
    r0 = min(rank * rows, H)
    r1 = min(r0 + rows, H)
    return r0, r1


def pack_band(out, n_band_rays, n_pad_rays):
    """[5 * n_pad] buffer: rgb (3n) | depth (n) | alphainv (n); the tail of a short band is zero."""
    dev = out['rgb_marched'].device
    buf = torch.zeros(5 * n_pad_rays, device=dev, dtype=torch.float32)
    buf[0:3 * n_band_rays] = out['rgb_marched'].reshape(-1)
    if 'depth' in out:
        buf[3 * n_pad_rays:3 * n_pad_rays + n_band_rays] = out['depth']
    buf[4 * n_pad_rays:4 * n_pad_rays + n_band_rays] = out['alphainv_last']
    return buf


def unpack_frame(gathered, H, W, world_size):
    """[world, 5 * n_pad] -> dict of full-frame tensors (padding rows dropped)."""
    rows = band_rows(H, world_size)
    n_pad = rows * W
    g = gathered.view(world_size, 5 * n_pad)
    rgb = g[:, :3 * n_pad].reshape(world_size * rows, W, 3)[:H]
    depth = g[:, 3 * n_pad:4 * n_pad].reshape(world_size * rows, W)[:H]
    ainv = g[:, 4 * n_pad:5 * n_pad].reshape(world_size * rows, W)[:H]
    return {'rgb_marched': rgb.reshape(H * W, 3), 'depth': depth.reshape(H * W), 'alphainv_last': ainv.reshape(H * W)}


class _DevMem:
    """A raw device allocation presented through ``__cuda_array_interface__`` (torch.as_tensor aliases it)."""

    def __init__(self, ptr, numel):
        self.__cuda_array_interface__ = {'shape': (int(numel),), 'typestr': '<f4', 'data': (int(ptr), False),
                                         'version': 2, 'strides': None}


class PeerBuffers:
    """``count`` fp32 device buffers of ``numel`` elements on every rank of ``group`` (one node, one process per GPU),
    each mapped into every other rank's address space: ``local[i]`` is this rank's buffer ``i`` as a tensor,
    ``ptrs[i][r]`` the device pointer under which THIS process reaches rank ``r``'s buffer ``i`` (``ptrs[i][rank]`` is the
    local one).  The kernels store results straight into the peers' buffers over NVLink (k4_render_rays_frames,
    k4_srnet_forward_roi_peers) -- SURVEY.md section 8e's "writing bands directly into peer-mapped output buffers" --
    and ``sync()`` orders the ranks: a one-element all-reduce enqueued behind the stores; once it has completed on a
    rank's stream, every rank's launch -- and with it every store into this rank's buffer -- has completed.

    The memory comes from the library (``k4_peer_alloc``: plain cudaMalloc, the caching allocator's blocks cannot be
    exported one by one) and is shared with CUDA IPC handles sent through ``all_gather_object``.  ``create`` is
    COLLECTIVE and returns ``None`` on every rank if any rank cannot allocate / export / map (not CUDA, ranks on
    different nodes, more than 8 ranks, ``K4_PEER=0``): the callers then use the all-gather path."""

    last_error = None          # why the last create() on this rank fell back (diagnostics)

    def __init__(self):
        self.local, self.ptrs, self._opened, self._owned = [], [], [], []

    @classmethod
    def create(cls, numel, device, group=None, count=2):
        from . import _lib
        device = torch.device(device)
        if not dist.is_initialized() or device.type != 'cuda' or os.environ.get('K4_PEER', '1') == '0':
            return None
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        if world < 2 or world > _lib.K4_MAX_PEERS:
            return None
        self = cls()
        self.group, self.world, self.rank, self.device, self.numel = group, world, rank, device, int(numel)
        ok, handles = 1, []
        with torch.cuda.device(device):
            try:
                if os.environ.get('K4_PEER_EAGER', '1') != '0':
                    _lib.check(_lib.lib.k4_peer_enable_all(), 'k4_peer_enable_all')
                for _ in range(count):
                    p = C.c_void_p()
                    _lib.check(_lib.lib.k4_peer_alloc(C.c_size_t(4 * self.numel), C.byref(p)), 'k4_peer_alloc')
                    self._owned.append(p.value)
                    h = C.create_string_buffer(64)
                    _lib.check(_lib.lib.k4_peer_export(C.c_void_p(p.value), h), 'k4_peer_export')
                    handles.append(h.raw)
            except Exception as e:
                ok, cls.last_error = 0, 'alloc/export: ' + repr(e)
            info = [None] * world
            dist.all_gather_object(info, (ok, handles, os.uname().nodename), group=group)
            ok = int(all(i[0] for i in info) and len({i[2] for i in info}) == 1)
            if ok:
                try:
                    for i in range(count):
                        row = []
                        for r in range(world):
                            if r == rank:
                                row.append(self._owned[i])
                                continue
                            q = C.c_void_p()
                            _lib.check(_lib.lib.k4_peer_open(info[r][1][i], C.byref(q)), 'k4_peer_open')
                            self._opened.append(q.value)
                            row.append(q.value)
                        self.ptrs.append(row)
                    self.local = [torch.as_tensor(_DevMem(p, self.numel), device=device) for p in self._owned]
                    if any(t.data_ptr() != p or not t.is_cuda for t, p in zip(self.local, self._owned)):
                        ok, cls.last_error = 0, 'torch.as_tensor copied the buffer instead of aliasing it'
                except Exception as e:
                    ok, cls.last_error = 0, 'open/alias: ' + repr(e)
            elif cls.last_error is None:
                cls.last_error = 'another rank failed or the ranks span nodes: ' + repr([(i[0], i[2]) for i in info])
            t = torch.tensor([ok], device=device, dtype=torch.int32)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
            if int(t.item()) == 0:
                self.close()
                return None
            self._flag = torch.zeros(1, device=device, dtype=torch.float32)
        return self

    def sync(self):
        """Stream-ordered barrier of the group (no host wait): behind it, the stores every rank issued before ITS
        ``sync()`` are complete."""
        dist.all_reduce(self._flag, group=self.group)

    def close(self):
        from . import _lib
        self.local = []
        for p in self._opened:
            _lib.lib.k4_peer_close(C.c_void_p(p))
        for p in self._owned:
            _lib.lib.k4_peer_free(C.c_void_p(p))
        self._opened, self._owned, self.ptrs = [], [], []


class FrameTarget:
    """Where one rank's rows of a block-cyclic frame go: ``frame_dst`` is the filled ``k4_frame_dst`` for
    ``render_rays(out=...)`` (every rank's image-order frame, the peers' reached through NVLink)."""

    def __init__(self, ptrs, rank, world, W, n_full):
        from . import _lib
        d = _lib.FrameDst()
        d.n_dst, d.rank, d.world, d.frame_w, d.n_full = len(ptrs), rank, world, W, n_full
        for i, p in enumerate(ptrs):
            d.d_frame[i] = p
        self.frame_dst = d


def frame_views(full, H, W, n_full):
    """dict views of an image-order frame buffer ``[rgb 3 n_full | depth n_full | alphainv n_full]``."""
    return {'rgb_marched': full[:3 * H * W].view(H * W, 3), 'depth': full[3 * n_full:3 * n_full + H * W],
            'alphainv_last': full[4 * n_full:4 * n_full + H * W]}


class CyclicFrame:
    """Cached plan + buffers of one rank for block-cyclic frame rendering (H x W over `world` ranks).

    ``render(make_rays, render_fn)`` = rays of the rank's rows only (``make_rays(rows) -> ro, rd, vd`` each [k*W,3]) ->
    fused march with ``render_fn(ro, rd, vd, (k, W), out)`` -> exchange -> every rank holds the frame in image order.

    Two exchanges.  PEER (default on the GPUs of one node): ``out`` is a :class:`FrameTarget` and the marcher stores
    every ray straight into the image-order frame of every rank (NVLink P2P stores from inside the kernel, overlapped
    with the march); a one-element all-reduce orders the ranks.  No band buffer, no all-gather, no transpose.  Two frame
    buffers alternate, so a rank that is one frame ahead never overwrites the frame another rank is still reading.
    GATHER (gloo / CPU tests, ``K4_PEER=0``, anything :class:`PeerBuffers` cannot map): ``out`` is a dict of views
    of the rank's packed send buffer (pad zeroed once), then ONE all-gather and the image-order transpose into a frame
    buffer allocated once."""

    def __init__(self, H, W, device, group=None):
        self.H, self.W, self.group = H, W, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.rows = cyclic_rows(H, self.rank, self.world).to(device=device, dtype=torch.int32).contiguous()
        self.k = int(self.rows.numel())
        self.n_band = self.k * W
        self.n_pad = cyclic_pad_rows(H, self.world) * W
        self.n_full = self.world * self.n_pad
        self.step = 0
        self.peers = PeerBuffers.create(5 * self.n_full, device, group, count=2) if self.world > 1 else None
        if self.peers is not None:
            self.targets = [FrameTarget(self.peers.ptrs[i], self.rank, self.world, W, self.n_full) for i in range(2)]
            return
        self.buf = torch.zeros(5 * self.n_pad, device=device, dtype=torch.float32)
        self.out = packed_band_views(self.buf, self.n_band, self.n_pad)
        self.gathered = torch.empty(self.world * 5 * self.n_pad, device=device, dtype=torch.float32) if self.world > 1 else self.buf
        # image-order frame, allocated once: a gather per step must not reach the allocator (a cudaMalloc inside a step
        # synchronises the device, and with NCCL's peer mappings in place it is slow)
        self.full = torch.empty(self.world * 5 * self.n_pad, device=device, dtype=torch.float32)

    def target(self):
        """``out=`` of this step's ``render_rays`` call: the peer frames of the step's parity, or the send-buffer views."""
        return self.targets[self.step & 1] if self.peers is not None else self.out

    def finish(self):
        """Complete the step's exchange; returns the frame (views, valid until the step after the next one in peer
        mode, until the next step in gather mode -- clone to keep one longer)."""
        if self.peers is not None:
            self.peers.sync()
            full = self.peers.local[self.step & 1]
            self.step += 1
            return frame_views(full, self.H, self.W, self.n_full)
        self.step += 1
        return self.gather()

    def gather(self):
        """(gather mode) all-gather + image-order transpose."""
        if self.world > 1:
            dist.all_gather_into_tensor(self.gathered, self.buf, group=self.group)
        return unpack_frame_cyclic(self.gathered, self.H, self.W, self.world, out=self.full)

    def render(self, make_rays, render_fn):
        if self.k > 0:
            ro, rd, vd = make_rays(self.rows)
            render_fn(ro, rd, vd, (self.k, self.W), self.target())
        return self.finish()


def render_frame_sharded(render_fn, rays_o, rays_d, viewdirs, H, W, group=None, gather=True, layout='cyclic'):
    """Render this rank's rows with ``render_fn(ro, rd, vd, image_hw) -> dict`` and all-gather the
    packed bands.  ``rays_*`` are the FULL frame ``[H*W, 3]`` (replicated or generated per rank); only
    this rank's rows are read.  ``layout``: 'cyclic' (8-row blocks dealt round-robin, load balanced,
    default) or 'bands' (contiguous).  Returns the full-frame dict on every rank (``gather=True``) or
    this rank's band dict.  (The device-resident drivers use :class:`CyclicFrame`, which generates only
    the rank's rays and lets the kernel write into the packed buffer.)"""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if layout == 'cyclic' and world > 1:
        rows = cyclic_rows(H, rank, world).to(rays_o.device)
        k = rows.numel()
        sel = lambda t: t.view(H, W, 3)[rows].reshape(-1, 3)
        if k > 0:
            out = render_fn(sel(rays_o), sel(rays_d), sel(viewdirs), (k, W))
        else:
            dev = rays_o.device
            out = {'rgb_marched': torch.zeros(0, 3, device=dev), 'depth': torch.zeros(0, device=dev),
                   'alphainv_last': torch.zeros(0, device=dev)}
        if not gather:
            return out
        n_pad = cyclic_pad_rows(H, world) * W
        buf = pack_band(out, k * W, n_pad)
        gathered = torch.empty(world * 5 * n_pad, device=buf.device, dtype=torch.float32)
        dist.all_gather_into_tensor(gathered, buf, group=group)
        return unpack_frame_cyclic(gathered, H, W, world)
    r0, r1 = band_range(H, rank, world)
    sl = slice(r0 * W, r1 * W)
    n_band = (r1 - r0) * W
    if n_band > 0:
        out = render_fn(rays_o[sl], rays_d[sl], viewdirs[sl], (r1 - r0, W))
    else:
        dev = rays_o.device
        out = {'rgb_marched': torch.zeros(0, 3, device=dev), 'depth': torch.zeros(0, device=dev),
               'alphainv_last': torch.zeros(0, device=dev)}
    if not gather or world == 1:
        return out
    n_pad = band_rows(H, world) * W
    buf = pack_band(out, n_band, n_pad)
    gathered = torch.empty(world * 5 * n_pad, device=buf.device, dtype=torch.float32)
    dist.all_gather_into_tensor(gathered, buf, group=group)
    return unpack_frame(gathered, H, W, world)


# ------------------------------------------------------------------------------------------------
# VC-Decoder sharding (SURVEY.md section 8e): by reference tile, tiles split into row parts with a
# recomputed halo when there are more ranks than tiles.
# ------------------------------------------------------------------------------------------------
def sr_units(height, width, tile_size, tile_pad, world_size, halo):
    """Work units of one x4 decode.  The reference's tile geometry (lib/sr_esrnet.py:467-527) is part
    of the result (the 10-pixel pad is far smaller than the receptive field), so the units are the
    reference tiles; with more ranks than tiles the tiles' OUTPUT rows are cut into row parts, each computed
    from its rows plus ``halo`` rows above and below, clipped to the PADDED TILE (beyond it the un-split tile
    sees zero padding too).  With ``halo`` >= the network's receptive radius every part reproduces the
    un-split tile's pixels exactly.

    Balance: the ranks are dealt to the tiles so that the most expensive part is as cheap as possible (a
    756-row frame has two 520-row and two 256-row padded tiles: 8 ranks -> 3 + 3 + 1 + 1, not 2 + 2 + 2 + 2),
    and the cuts inside a tile equalise the parts' cost, where a part costs its kept rows + its pad rows +
    ~halo/2 rows per cut side (every layer only computes the rows inside the remaining receptive field of the
    kept rows, SFTNet.forward_roi, so a cut costs half the halo on average).

    Returns a list of dicts: ``src`` = (y0, y1, x0, x1) input crop in LR pixels, ``keep`` = (ky, kx)
    offset of the kept block inside the unit's output in LR pixels, ``dst`` = (y0, y1, x0, x1) LR
    rect of the kept block in the image, ``cost`` = the model above (LR pixels)."""
    import math
    tiles_x = math.ceil(width / tile_size)
    tiles_y = math.ceil(height / tile_size)
    tiles = []
    for ty in range(tiles_y):
        for tx in range(tiles_x):
            x0, y0 = tx * tile_size, ty * tile_size
            x1, y1 = min(x0 + tile_size, width), min(y0 + tile_size, height)
            x0p, x1p = max(x0 - tile_pad, 0), min(x1 + tile_pad, width)
            y0p, y1p = max(y0 - tile_pad, 0), min(y1 + tile_pad, height)
            tiles.append((y0, y1, x0, x1, y0p, y1p, x0p, x1p))
    cut_cost = halo / 2.0

    def parts_of(t, n):
        """Row boundaries of tile t cut into n parts of equal modelled cost; list of (ya, yb, overhead rows)."""
        y0, y1, _, _, y0p, y1p, _, _ = t
        rows = y1 - y0
        n = max(1, min(n, rows))
        over = [((y0 - y0p) if k == 0 else cut_cost) + ((y1p - y1) if k == n - 1 else cut_cost) for k in range(n)]
        target = (rows + sum(over)) / n
        want = [max(1.0, target - o) for o in over]
        scale = rows / sum(want)
        edges, acc = [y0], 0.0
        for k in range(n - 1):
            acc += want[k] * scale
            edges.append(min(max(int(round(y0 + acc)), edges[-1] + 1), y1 - (n - 1 - k)))
        edges.append(y1)
        return [(edges[k], edges[k + 1], over[k]) for k in range(n)]

    def worst(t, n):
        w = t[7] - t[6]
        return max((yb - ya + o) * w for ya, yb, o in parts_of(t, n))

    def split_to(total):
        sp = [1] * len(tiles)
        while sum(sp) < total:
            cand = [i for i in range(len(tiles)) if sp[i] < tiles[i][1] - tiles[i][0]]
            if not cand:
                break
            i = max(cand, key=lambda i: worst(tiles[i], sp[i]))
            sp[i] += 1
        return sp

    def max_load(sp):
        """Largest per-rank cost after longest-first assignment; every unit also pays a fixed ~24 rows of launch /
        fill / drain overhead (~120 kernels of ~10 us)."""
        costs = sorted(((yb - ya + o + 24.0) * (t[7] - t[6]) for t, n in zip(tiles, sp) for ya, yb, o in parts_of(t, n)), reverse=True)
        load = [0.0] * world_size
        for c in costs:
            load[load.index(min(load))] += c
        return max(load)

    # as many units as ranks is the natural choice; a few more can balance better when tiles differ in size
    # (4 ranks, tiles of 520/520/256/256 rows: 8 units of ~230 rows pack to 483 per rank, 4 whole tiles to 520)
    splits = min((split_to(total) for total in range(max(world_size, 1), 3 * max(world_size, 1) + 1)),
                 key=lambda sp: (max_load(sp), sum(sp))) if world_size > 1 else [1] * len(tiles)
    units = []
    for t, n in zip(tiles, splits):
        y0, y1, x0, x1, y0p, y1p, x0p, x1p = t
        pp = parts_of(t, n)
        for k, (ya, yb, o) in enumerate(pp):
            sa = y0p if k == 0 else max(ya - halo, y0p)
            sb = y1p if k == len(pp) - 1 else min(yb + halo, y1p)
            units.append({'src': (sa, sb, x0p, x1p), 'keep': (ya - sa, x0 - x0p), 'dst': (ya, yb, x0, x1),
                          'cost': (yb - ya + o) * (x1p - x0p)})
    return units


def sr_assign(units, world_size):
    """Units of each rank: longest-processing-time first (one unit per rank when there are as many units as ranks)."""
    order = sorted(range(len(units)), key=lambda i: (-units[i]['cost'], i))
    load = [0.0] * world_size
    mine = [[] for _ in range(world_size)]
    for i in order:
        r = min(range(world_size), key=lambda r: load[r])
        load[r] += units[i]['cost']
        mine[r].append(i)
    return [sorted(m) for m in mine]


_SR_PLANS = {}


def sr_plan(H, W, tile_size, tile_pad, world, halo):
    """(units, assign) of :func:`sr_units` / :func:`sr_assign`, computed once per geometry: the balancing search is a few
    milliseconds of Python at 8 ranks -- as long as the whole 8-GPU frame -- and must not run per frame."""
    key = (int(H), int(W), int(tile_size), int(tile_pad), int(world), int(halo))
    plan = _SR_PLANS.get(key)
    if plan is None:
        units = sr_units(*key)
        plan = _SR_PLANS[key] = (units, sr_assign(units, key[4]))
    return plan


def sr_decode_sharded(net_fn, img, cond, tile_size, tile_pad=10, scale=4, halo=80, group=None, net_units_fn=None,
                      peers=None):
    """x`scale` decode of ``img [1,C,H,W]`` / ``cond [num_cond,H,W]`` (full frame on every rank; ``num_cond`` 1 for the
    depth condition, 63 / 64 for the view-conditioned decoder) with the units
    of :func:`sr_units` dealt round-robin over the ranks and ONE all-gather of the packed output
    blocks.  ``net_fn(img_crop, cond_crop[1,num_cond,h,w]) -> [1,C,scale*h,scale*w]`` is the decoder
    (``SFTNet.forward``); ``net_units_fn(jobs)`` with ``jobs = [(img_crop, cond_crop, (y0,y1,x0,x1), out[C,.,.]), ...]``
    (``SFTNet.run_units``), when given, writes every unit's kept block straight into the packed send buffer, lets every
    layer skip the rows outside the kept block's remaining receptive field and overlaps a rank's units on two
    streams.  Every rank returns the full
    ``[1,C,scale*H,scale*W]`` frame.  ``peers`` (a :class:`PeerBuffers` of ``C*scale*H*scale*W`` elements, with
    ``net_units_fn``): no packed buffer, no all-gather, no assembly -- every unit's kept block is stored by the
    decoder's last kernel into the frame of EVERY rank (its own and, over NVLink, the peers'), then ``peers.sync()``."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    _, C, H, W = img.shape
    s = scale
    units, assign = sr_plan(H, W, tile_size, tile_pad, world, halo)
    size = lambda u: C * (u['dst'][1] - u['dst'][0]) * (u['dst'][3] - u['dst'][2]) * s * s
    if peers is not None and net_units_fn is not None and world > 1:
        par = peers.__dict__.setdefault('_step', 0) & 1
        peers._step += 1
        output = peers.local[par].view(1, C, H * s, W * s)
        cond4 = cond.unsqueeze(0)
        jobs = []
        for u in (units[i] for i in assign[rank]):
            sa, sb, xa, xb = u['src']
            ky, kx = u['keep']
            y0, y1, x0, x1 = u['dst']
            blk = output[0, :, y0 * s:y1 * s, x0 * s:x1 * s]
            off = 4 * (blk.storage_offset() - output.storage_offset())          # same window in every rank's frame
            extra = [peers.ptrs[par][r] + off for r in range(world) if r != rank]
            jobs.append((img[:, :, sa:sb, xa:xb], cond4[:, :, sa:sb, xa:xb], (ky, ky + y1 - y0, kx, kx + x1 - x0), blk, extra))
        if jobs:
            net_units_fn(jobs)
        peers.sync()
        return output
    per_rank = [sum(size(units[i]) for i in assign[r]) for r in range(world)]
    n_pad = max(per_rank) if per_rank else 0
    buf = torch.empty(n_pad, device=img.device, dtype=img.dtype)
    off = 0
    cond4 = cond.unsqueeze(0)
    jobs = []
    for u in (units[i] for i in assign[rank]):
        sa, sb, xa, xb = u['src']
        ky, kx = u['keep']
        y0, y1, x0, x1 = u['dst']
        n = size(u)
        blk = buf[off:off + n].view(C, (y1 - y0) * s, (x1 - x0) * s)
        if net_units_fn is not None:
            jobs.append((img[:, :, sa:sb, xa:xb], cond4[:, :, sa:sb, xa:xb], (ky, ky + y1 - y0, kx, kx + x1 - x0), blk))
        else:
            out = net_fn(img[:, :, sa:sb, xa:xb], cond4[:, :, sa:sb, xa:xb])
            blk.copy_(out[0, :, ky * s:(ky + y1 - y0) * s, kx * s:(kx + x1 - x0) * s])
        off += n
    if jobs:
        net_units_fn(jobs)
    if world > 1:
        gathered = torch.empty(world * n_pad, device=img.device, dtype=img.dtype)
        dist.all_gather_into_tensor(gathered, buf, group=group)
    else:
        gathered = buf
    g = gathered.view(world, n_pad)
    output = torch.empty((1, C, H * s, W * s), device=img.device, dtype=img.dtype)
    for r in range(world):
        off = 0
        for u in (units[i] for i in assign[r]):
            y0, y1, x0, x1 = u['dst']
            n = size(u)
            output[0, :, y0 * s:y1 * s, x0 * s:x1 * s] = g[r, off:off + n].view(C, (y1 - y0) * s, (x1 - x0) * s)
            off += n
    return output
