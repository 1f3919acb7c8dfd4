"""SFTNet (the VC-Decoder) with the reference's constructor, parameter names and call contract
(lib/sr_esrnet.py:400-527), executed by the wgmma convolution pipeline of libk4nerf.so
(csrc/k4_sr.cu).  The module tree below only OWNS the parameters (so reference checkpoints and
``pretrained/RealESRNet_x4plus.pth`` load with the same keys, ``strict=False`` as run_sr.py:663);
no torch op runs in ``forward``."""
import ctypes as C
import math
from copy import deepcopy
from fractions import Fraction

import torch
from torch import nn

from . import _lib
from ._scene import require_cuda


class SFTLayer(nn.Module):
    def __init__(self, num_feat=64, num_grow_ch=32):
        super().__init__()
        self.SFT_scale_conv0 = nn.Conv2d(num_grow_ch, num_grow_ch, 1)
        self.SFT_scale_conv1 = nn.Conv2d(num_grow_ch, num_feat, 1)
        self.SFT_shift_conv0 = nn.Conv2d(num_grow_ch, num_grow_ch, 1)
        self.SFT_shift_conv1 = nn.Conv2d(num_grow_ch, num_feat, 1)

    def convs(self):
        return [self.SFT_scale_conv0, self.SFT_scale_conv1, self.SFT_shift_conv0, self.SFT_shift_conv1]


class ResidualDenseBlock_SFT(nn.Module):
    def __init__(self, num_feat=64, num_grow_ch=32):
        super().__init__()
        self.conv1 = nn.Conv2d(num_feat, num_grow_ch, 3, 1, 1)
        self.conv2 = nn.Conv2d(num_feat + num_grow_ch, num_grow_ch, 3, 1, 1)
        self.conv3 = nn.Conv2d(num_feat + 2 * num_grow_ch, num_grow_ch, 3, 1, 1)
        self.conv4 = nn.Conv2d(num_feat + 3 * num_grow_ch, num_grow_ch, 3, 1, 1)
        self.conv5 = nn.Conv2d(num_feat + 4 * num_grow_ch, num_feat, 3, 1, 1)
        self.sft0 = SFTLayer(num_feat, num_grow_ch)
        self.sft1 = SFTLayer(num_grow_ch, num_grow_ch)
        for c in (self.conv1, self.conv2, self.conv3, self.conv4, self.conv5):   # default_init_weights(..., 0.1)
            nn.init.kaiming_normal_(c.weight)
            c.weight.data *= 0.1
            c.bias.data.zero_()


class RRDB_SFT(nn.Module):
    def __init__(self, num_feat, num_grow_ch=32):
        super().__init__()
        self.rdb1 = ResidualDenseBlock_SFT(num_feat, num_grow_ch)
        self.rdb2 = ResidualDenseBlock_SFT(num_feat, num_grow_ch)
        self.rdb3 = ResidualDenseBlock_SFT(num_feat, num_grow_ch)
        self.sft0 = SFTLayer(num_feat, num_grow_ch)


def sft_condition(num_cond, depth, viewdirs, H, W):
    """The SFT condition ``[num_cond, H, W]`` of an H x W LR frame, the one run_sr.py selects with
    ``cfg.fine_model_and_render.num_cond`` before every decoder call:

    * 1: the marched depth (run_sr.py:895-898, :1365-1367);
    * 63: the view-direction embedding at every pixel, ``[v, sin(v * 2^i), cos(v * 2^i)]``, i = 0..9, v = the pixel's
      normalised ``viewdirs``; the 30 sin (cos) channels ordered by direction axis first, frequency second
      (run_sr.py:899-904, :1368-1373);
    * 64: depth as channel 0, then the 63 channels above -- the training path's ``torch.cat((depth, emb), 1)``
      (run_sr.py:905-912).  The reference's validation, test and video paths fail for 64 (they index a 3-D depth with
      four indices, run_sr.py:1376, or concatenate 3-D with 4-D tensors), so the training path defines it.

    ``depth``: ``H*W`` values (any shape of that size), ``viewdirs``: ``[H*W, 3]`` (or ``[H, W, 3]``), on one device.
    The embedding uses run_sr.py's own torch expressions, so on the same device its values equal the reference's bit for
    bit.  Other ``num_cond`` values raise: the reference's driver defines no other condition."""
    H, W = int(H), int(W)
    if num_cond not in (1, 63, 64):
        raise ValueError(f'run_sr.py defines the SFT condition for num_cond 1, 63 and 64 only, got {num_cond!r}')
    if num_cond == 1:
        return depth.reshape(1, H, W)
    viewdirs = viewdirs.reshape(H * W, 3)
    viewfreq = torch.FloatTensor([(2**i) for i in range(10)]).to(viewdirs.device)
    emb = (viewdirs.unsqueeze(-1) * viewfreq).flatten(-2)
    emb = torch.cat([viewdirs, emb.sin(), emb.cos()], -1)
    emb = emb.reshape(H, W, -1).movedim(-1, 0)
    if num_cond == 63:
        return emb.contiguous()
    return torch.cat((depth.reshape(1, H, W).to(emb.dtype), emb), 0)


class _NetHandle:
    def __init__(self, ptr, fingerprint):
        self.ptr, self.fingerprint = ptr, fingerprint

    def __del__(self):
        try:
            if self.ptr:
                _lib.lib.k4_srnet_destroy(self.ptr)
                self.ptr = None
        except Exception:
            pass


class SFTNet(nn.Module):
    def __init__(self, n_in_colors, scale, num_feat=64, num_block=5, num_grow_ch=32, num_cond=1, dswise=False):
        super().__init__()
        if int(num_cond) != num_cond or num_cond < 1:
            raise ValueError(f'num_cond must be a positive integer (the condition channels of CondNet.0), got {num_cond!r}')
        num_cond = int(num_cond)
        if dswise or n_in_colors != 3 or scale not in (1, 4) or num_feat != 64 or num_grow_ch != 32 or num_cond > 64:
            raise NotImplementedError('k4nerf builds the shipped VC-Decoders: SFTNet(3, 4, 64, n, 32, c) (run_sr.py:1353) and '
                                      'SFTNet(3, 1, 64, n, 32, c) (the 1x configs) with a condition of c = 1..64 channels')
        self.scale = scale
        self.num_cond = num_cond
        self.dswise = dswise
        self.conv_first = nn.Conv2d(n_in_colors, num_feat, 3, 1, 1)
        self.body = nn.Sequential(*[RRDB_SFT(num_feat=num_feat, num_grow_ch=num_grow_ch) for _ in range(num_block)])
        self.conv_body = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        if scale == 4:                     # x1 registers no upsampling convs (lib/sr_esrnet.py:430-433)
            self.conv_up1 = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
            self.conv_up2 = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_hr = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_last = nn.Conv2d(num_feat, 3, 3, 1, 1)
        self.sftbody = SFTLayer(num_feat, num_grow_ch)
        self.CondNet = nn.Sequential(
            nn.Conv2d(num_cond, 64, 3, 1, 1), nn.LeakyReLU(0.2, True),
            nn.Conv2d(64, 64, 1), nn.LeakyReLU(0.2, True),
            nn.Conv2d(64, 64, 1), nn.LeakyReLU(0.2, True),
            nn.Conv2d(64, 32, 1))
        self._cfg = (n_in_colors, scale, num_feat, num_block, num_grow_ch, num_cond)

    # -- parameter order of include/k4nerf.h (k4_srnet_desc) ---------------------------------------
    def _ordered_convs(self):
        cs = [self.conv_first, self.CondNet[0], self.CondNet[2], self.CondNet[4], self.CondNet[6]]
        for blk in self.body:
            for rdb in (blk.rdb1, blk.rdb2, blk.rdb3):
                cs += [rdb.conv1, rdb.conv2, rdb.conv3, rdb.conv4, rdb.conv5] + rdb.sft0.convs() + rdb.sft1.convs()
            cs += blk.sft0.convs()
        cs += self.sftbody.convs() + [self.conv_body]
        if self.scale == 4:
            cs += [self.conv_up1, self.conv_up2]
        cs += [self.conv_hr, self.conv_last]
        return cs

    def _get_net(self):
        params = [t for c in self._ordered_convs() for t in (c.weight, c.bias)]     # live Parameters: replaced ones are seen
        fp = tuple([(t.data_ptr(), t._version) for t in params])
        h = getattr(self, '_k4_net', None)
        if h is not None and h.fingerprint == fp:
            return h
        require_cuda(*params)
        dev = params[0].device
        keep = [t.detach().to(torch.float32).contiguous() for t in params]
        arr = (C.c_void_p * len(keep))(*[t.data_ptr() for t in keep])
        d = _lib.SrnetDesc()
        d.n_in_colors, d.scale, d.num_feat, d.num_block, d.num_grow_ch, d.num_cond = self._cfg
        d.n_params = len(keep)
        d.h_params = C.cast(arr, C.POINTER(C.c_void_p))
        out = C.c_void_p()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            _lib.check(_lib.lib.k4_srnet_create(C.byref(d), C.c_void_p(stream.cuda_stream), C.byref(out)), 'k4_srnet_create')
            stream.synchronize()
        h = _NetHandle(out.value, fp)
        object.__setattr__(self, '_k4_net', h)
        return h

    def _workspace(self, nbytes, dev, slot=0):
        pool = self.__dict__.setdefault('_k4_ws_pool', {})
        ws = pool.get((dev, slot))
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(int(nbytes), device=dev, dtype=torch.uint8)
            pool[(dev, slot)] = ws
        return ws

    @torch.no_grad()
    def forward_roi(self, x, cond, keep, out, ws_slot=0, extra=None):
        """The output pixels (``s = self.scale`` per LR pixel and axis) of LR block ``keep = (y0, y1, x0, x1)`` of tile
        ``x [1,3,h,w]`` / ``cond [1,num_cond,h,w]`` written into ``out``: a ``[3, s(y1-y0), s(x1-x0)]`` fp32 CUDA view with unit
        stride along x (typically a window of the frame).  Same values as ``forward(x, cond)[0, :, s*y0:s*y1, s*x0:s*x1]``;
        every layer computes only the rows inside the
        remaining receptive field of the kept rows (k4_srnet_forward_roi).  Runs on the current stream.  ``extra``: device
        pointers (ints) of the same window in other ranks' peer-mapped frames -- the last convolution stores the block there
        too (k4_srnet_forward_roi_peers)."""
        require_cuda(x, cond, out)
        self._check_inputs(x, cond)
        h, w = int(x.shape[2]), int(x.shape[3])
        y0, y1, x0, x1 = [int(v) for v in keep]
        s = self.scale
        assert out.dtype == torch.float32 and tuple(out.shape) == (3, (y1 - y0) * s, (x1 - x0) * s) and out.stride(2) == 1
        net = self._get_net()
        dev = x.device
        x = x.to(torch.float32).contiguous()
        cond = cond.to(torch.float32).contiguous()
        nbytes = int(_lib.lib.k4_srnet_workspace_bytes(net.ptr, h, w))
        ws = self._workspace(nbytes, dev, ws_slot)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            if extra:
                arr = (C.c_void_p * len(extra))(*[int(e) for e in extra])
                _lib.check(_lib.lib.k4_srnet_forward_roi_peers(net.ptr, x.data_ptr(), cond.data_ptr(), h, w, y0, y1, x0, x1,
                                                               out.data_ptr(), int(out.stride(0)), int(out.stride(1)),
                                                               len(extra), arr, ws.data_ptr(), ws.numel(),
                                                               C.c_void_p(stream)), 'k4_srnet_forward_roi_peers')
            else:
                _lib.check(_lib.lib.k4_srnet_forward_roi(net.ptr, x.data_ptr(), cond.data_ptr(), h, w, y0, y1, x0, x1,
                                                         out.data_ptr(), int(out.stride(0)), int(out.stride(1)),
                                                         ws.data_ptr(), ws.numel(), C.c_void_p(stream)), 'k4_srnet_forward_roi')
        return out

    @torch.no_grad()
    def run_units(self, jobs, streams=2):
        """``forward_roi`` for a list of independent jobs ``(x_crop [1,3,h,w], cond_crop [1,num_cond,h,w], keep, out_view[, extra])``
        dealt (largest first) to
        ``streams`` CUDA streams with a workspace each; returns when the current stream has been made to wait for all of
        them.  Independent units overlap each other's launch / fill / drain phases (~120 kernels per unit)."""
        if not jobs:
            return
        for job in jobs:
            self._check_inputs(job[0], job[1])
        dev = jobs[0][0].device
        n_streams = max(1, min(int(streams), len(jobs)))
        cur = torch.cuda.current_stream(dev)
        side = self.__dict__.setdefault('_k4_streams', {})
        pool = [cur] + [side.setdefault((dev, i), torch.cuda.Stream(dev)) for i in range(1, n_streams)]
        if n_streams > 1:
            ready = torch.cuda.Event()
            ready.record(cur)
        order = sorted(range(len(jobs)), key=lambda i: -jobs[i][0].shape[2] * jobs[i][0].shape[3])
        load = [0] * n_streams
        used = set()
        for i in order:
            x, c, keep, out = jobs[i][:4]
            extra = jobs[i][4] if len(jobs[i]) > 4 else None
            k = min(range(n_streams), key=lambda j: load[j])
            load[k] += x.shape[2] * x.shape[3]
            st = pool[k]
            with torch.cuda.stream(st):
                if k > 0 and k not in used:
                    st.wait_event(ready)
                used.add(k)
                xt, ct = x.contiguous(), c.contiguous()
                self.forward_roi(xt, ct, keep, out, ws_slot=k, extra=extra)
                if k > 0:
                    xt.record_stream(st); ct.record_stream(st)
        for k in sorted(used - {0}):
            done = torch.cuda.Event()
            done.record(pool[k])
            cur.wait_event(done)

    @torch.no_grad()
    def forward(self, x, cond, fea=None):
        """x [1,3,h,w], cond [1,num_cond,h,w] (CUDA, fp32) -> [1,3,s*h,s*w], s = self.scale  (lib/sr_esrnet.py:446-465)."""
        if fea is not None:
            raise NotImplementedError('the `fea` branch needs conv_prefea (n_in_colors > 3), not in the shipped config')
        require_cuda(x, cond)
        self._check_inputs(x, cond)
        h, w = int(x.shape[2]), int(x.shape[3])
        out = torch.empty((1, 3, h * self.scale, w * self.scale), device=x.device, dtype=torch.float32)
        self.forward_roi(x, cond, (0, h, 0, w), out[0])
        return out

    @torch.no_grad()
    def tile_process(self, img, cond, tile_size, tile_pad=10, to_cpu=True, streams=2):
        """SFTNet.tile_process (lib/sr_esrnet.py:467-527): same tile geometry (the 10-pixel pad is far
        smaller than the receptive field, so the tiling is part of the result).  Every tile's kept block is
        written by the last convolution straight into the frame (no crop copies), the frame is assembled on
        the device and moved to the CPU once (the reference copies every tile), and the tiles are dealt to
        ``streams`` CUDA streams with a workspace each: the tiles are independent, so the launch / fill /
        drain phases of one tile's ~120 kernels overlap the other tile's work.

        ``img [1,3,H,W]``, ``cond [num_cond,H,W]``: the condition is unsqueezed inside, as the reference does (:474).  A 4-D
        condition raises (the reference would slice the wrong axes of it)."""
        batch, channel, height, width = img.shape
        assert batch == 1
        self._check_frame_cond(cond, height, width)
        cond = cond.unsqueeze(0)
        s = self.scale
        dev = img.device
        output = torch.empty((batch, channel, height * s, width * s), device=dev, dtype=torch.float32)
        tiles_x = math.ceil(width / tile_size)
        tiles_y = math.ceil(height / tile_size)
        tiles = []
        for y in range(tiles_y):
            for x in range(tiles_x):
                x0, y0 = x * tile_size, y * tile_size
                x1, y1 = min(x0 + tile_size, width), min(y0 + tile_size, height)
                x0p, x1p = max(x0 - tile_pad, 0), min(x1 + tile_pad, width)
                y0p, y1p = max(y0 - tile_pad, 0), min(y1 + tile_pad, height)
                tiles.append((y0p, y1p, x0p, x1p, y0, y1, x0, x1))
        jobs = [(img[:, :, y0p:y1p, x0p:x1p], cond[:, :, y0p:y1p, x0p:x1p], (y0 - y0p, y1 - y0p, x0 - x0p, x1 - x0p),
                 output[0, :, y0 * s:y1 * s, x0 * s:x1 * s]) for (y0p, y1p, x0p, x1p, y0, y1, x0, x1) in tiles]
        self.run_units(jobs, streams)
        return output.to('cpu') if to_cpu else output

    def _check_inputs(self, x, cond):
        """A tile: x [1,3,h,w] and cond [1,num_cond,h,w]."""
        assert x.dim() == 4 and x.shape[0] == 1 and x.shape[1] == 3, f'x must be [1,3,h,w], got {tuple(x.shape)}'
        if cond.dim() != 4 or cond.shape[0] != 1 or cond.shape[1] != self.num_cond or cond.shape[2:] != x.shape[2:]:
            raise ValueError(f'cond must be [1,{self.num_cond},{x.shape[2]},{x.shape[3]}] (num_cond = {self.num_cond}), '
                             f'got {tuple(cond.shape)}')

    def _check_frame_cond(self, cond, height, width):
        """A frame's condition for tile_process: [num_cond,H,W], the reference's contract (lib/sr_esrnet.py:474)."""
        if cond.dim() != 3 or tuple(cond.shape) != (self.num_cond, height, width):
            raise ValueError(f'tile_process takes cond [num_cond,H,W] = [{self.num_cond},{height},{width}] and unsqueezes it '
                             f'itself (lib/sr_esrnet.py:474), got {tuple(cond.shape)}')

    def receptive_halo(self):
        """LR rows a decoded pixel can depend on above/below it: conv_first/CondNet.0 (1) + 15 3x3 convs
        per RRDB_SFT + conv_body (1) + the tail, rounded up to an even count.  The tail is the 3x3 convs behind
        conv_body, each 1 row at its own resolution: at x4 conv_up1 (1/2 LR row) and conv_up2, conv_hr, conv_last
        (1/4 each), 5/4 -> 2 LR rows; at x1 conv_hr + conv_last at LR, 2 rows.  So the halo is 80 for 5 blocks at
        either scale.  Row parts of a tile cut with this halo reproduce the un-split tile exactly (dist.sr_units)."""
        res = ([2, 4] if self.scale == 4 else []) + [self.scale, self.scale]     # resolution factor of each tail conv
        tail = math.ceil(sum(Fraction(1, f) for f in res))
        r = 1 + 15 * len(self.body) + 1 + tail
        return r + (r & 1)

    def tile_process_sharded(self, img, cond, tile_size, tile_pad=10, group=None):
        """tile_process across the ranks of ``group`` (SURVEY.md section 8e): reference tiles (split into
        row parts with a recomputed halo when ranks outnumber tiles) dealt to the ranks; every rank returns the same
        full frame as single-GPU ``tile_process`` (device resident).  On the GPUs of one node every unit's last
        convolution stores its kept block straight into every rank's frame (peer-mapped, :class:`k4nerf.dist.PeerBuffers`;
        two frames alternate, the returned one is valid until the call after the next one); otherwise one all-gather of
        the packed blocks + assembly.  ``cond [num_cond,H,W]`` as in :meth:`tile_process`."""
        from . import dist as kdist
        batch, channel, height, width = img.shape
        self._check_frame_cond(cond, height, width)
        peers = None
        if img.is_cuda and kdist.dist.is_initialized():
            cache = self.__dict__.setdefault('_k4_peer_frames', {})
            key = (channel, height, width, img.device, id(group))
            if key not in cache:       # collective: every rank decodes the same frame shape
                cache[key] = kdist.PeerBuffers.create(channel * height * width * self.scale ** 2, img.device, group, count=2)
            peers = cache[key]
        return kdist.sr_decode_sharded(lambda x, c: self(x, c), img, cond, tile_size, tile_pad, self.scale,
                                       self.receptive_halo(), group,
                                       net_units_fn=lambda jobs: self.run_units(jobs, streams=2), peers=peers)

    def load_network(self, load_path, device, strict=True, param_key='params_ema'):
        """lib/sr_esrnet.py:529-554 (keys may carry a 'module.' prefix; mismatching sizes are skipped
        when strict=False)."""
        load_net = torch.load(load_path, map_location=device, weights_only=False)
        if param_key is not None:
            if param_key not in load_net and 'params' in load_net:
                param_key = 'params'
            load_net = load_net[param_key]
        for k, v in deepcopy(load_net).items():
            if k.startswith('module.'):
                load_net[k[7:]] = v
                load_net.pop(k)
        if not strict:
            cur = self.state_dict()
            for k in list(load_net):
                if k in cur and cur[k].size() != load_net[k].size():
                    load_net[k + '.ignore'] = load_net.pop(k)
        self.load_state_dict(load_net, strict=strict)

    def save_network(self, save_root, net_label, current_iter, param_key='params'):
        """lib/sr_esrnet.py:589-622: ``<save_root>/<net_label>_<iter|latest>.pth`` holding ``{param_key: state_dict}`` with
        CPU tensors and any 'module.' prefix dropped -- the file ``load_network`` (and the reference's) reads back.  Like
        the reference, a failing write is retried three times and then reported, not raised."""
        import os
        import time
        name = 'latest' if current_iter == -1 else current_iter
        save_path = os.path.join(save_root, f'{net_label}_{name}.pth')
        state = {}
        for key, param in self.state_dict().items():
            state[key[7:] if key.startswith('module.') else key] = param.detach().cpu()
        for attempt in range(3):
            try:
                torch.save({param_key: state}, save_path)
                return save_path
            except Exception as e:       # noqa: BLE001 -- the reference swallows every error here
                print(f'Save model error: {e}, remaining retry times: {2 - attempt}')
                time.sleep(1)
        print(f'Still cannot save {save_path}. Just ignore it.')
        return None
