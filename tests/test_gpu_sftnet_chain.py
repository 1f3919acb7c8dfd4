"""GPU: the VC-Decoder's real forward layer by layer, in place, against float64, and tile_process's tiling bit for bit.

k4_testing_srnet_forward_upto runs k4_srnet_forward_roi and returns after its first k steps (one step: a layer as the
forward enqueues it).  Each case poisons the workspace with 0xFF bytes (fp16 / fp32 NaN) before every prefix run and keeps
the snapshots after k - 1 and after k steps.  Step k must be the layer that the reference module's structure puts
there.  Its operands are read from snapshot k - 1, where the test's own workspace plan puts them.  The layer is then
recomputed in float64 with the references and element bounds of test_gpu_sr_layers.py and test_gpu_sftnet_cond.py,
and checked against snapshot k:
  * every element it must produce, on the rows the layers after it still need, is finite and within its bound;
  * every byte outside its declared output (buffer, channels and rows) is unchanged.
The layer order comes from oracle/sftnet.py (sftnet_forward, rrdb_sft, rdb_sft).  With SFT fused, each SFT layer runs
in the epilogue of the convolution that produces its input (DESIGN.md section 3.4).  The rows each layer must produce
come from the receptive fields of the 3x3 convolutions behind it in that structure, not from the library's row
arithmetic.  Any read of a row that no layer wrote in this call is therefore a NaN in a checked row.
"""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import k4nerf
from k4nerf import _lib
from oracle import sftnet
from test_gpu_sr_layers import (FP16_MAX, FP32, FP32_EPS, MMA, RES_SCALE, conv_ref, sft_ref, sft_ref32, ulp16,
                                condnet_ref as condnet_ref_depth)
from test_gpu_sftnet_cond import condnet_ref as condnet_ref_wide
from test_sftnet_cond import frame_condition
from test_sftnet_x1 import x1_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUM_BLOCK = 5


# ------------------------------------------------------------------------------------------------
# the reference structure
# ------------------------------------------------------------------------------------------------
def reference_ops(num_block, scale):
    """The reference module's layers in forward order: (step, output tensor, [(input tensor, how it is read)]) with step
    = (kind, RRDB, dense block, conv) and `how` 'conv' (a 3x3 convolution), 'up' (nearest x2, then a 3x3 convolution)
    or 'pw' (per pixel).  The trunk entering RRDB i is also its residual (rrdb_sft); a dense block's input is its
    residual (rdb_sft)."""
    ops = [(('input', -1, -1, -1), 'x', []), (('condnet', -1, -1, -1), 'cond', []),
           (('conv_first', -1, -1, -1), 'feat', [('x', 'conv')])]
    x = 'feat'
    for i in range(num_block):
        x_in = x
        for j in range(3):
            r = f'{i}.{j}'
            ops.append((('sft0', i, j, -1), f'xc0.{r}', [(x, 'pw'), ('cond', 'pw')]))
            cat = [f'xc0.{r}']
            for c in range(4):
                ops.append((('rdb_conv', i, j, c), f'x{c + 1}.{r}', [(t, 'conv') for t in cat]))
                cat.append(f'x{c + 1}.{r}')
            ops.append((('sft1', i, j, -1), f'xc1.{r}', [(f'x4.{r}', 'pw'), ('cond', 'pw')]))
            ops.append((('rdb_conv', i, j, 4), f'y.{r}', [(t, 'conv') for t in cat[:4] + [f'xc1.{r}']] + [(x, 'pw')]))
            x = f'y.{r}'
        ops.append((('sft_rrdb', i, -1, -1), f'rrdb.{i}', [(x, 'pw'), ('cond', 'pw'), (x_in, 'pw')]))
        x = f'rrdb.{i}'
    ops.append((('sft_body', -1, -1, -1), 'sbody', [(x, 'pw'), ('cond', 'pw')]))
    ops.append((('conv_body', -1, -1, -1), 'bf', [('sbody', 'conv'), ('feat', 'pw')]))
    src = 'bf'
    if scale == 4:
        ops += [(('up1', -1, -1, -1), 'up1', [('bf', 'up')]), (('up2', -1, -1, -1), 'up2', [('up1', 'up')])]
        src = 'up2'
    ops.append((('hr', -1, -1, -1), 'hr', [(src, 'conv')]))
    ops.append((('last', -1, -1, -1), 'out', [('hr', 'conv')]))
    return ops


def resolution(t, scale):
    return {'up1': 2, 'up2': 4, 'hr': scale, 'out': scale}.get(t, 1)


def steps_of(ops, fused):
    """The launch sequence: one step per layer, or with SFT fused, every SFT layer folded into the step that produced
    its input (so conv_first, conv4 and conv5 carry SFT epilogues).  Returns [(descriptor, [ops])]."""
    groups, producer = [], {}
    for op in ops:
        (kind, *_), out, ins = op
        if fused and kind.startswith('sft'):
            g = producer[ins[0][0]]
            g.append(op)
        else:
            g = [op]
            groups.append(g)
        producer[out] = g
    return [(g[0][0] + (int(len(g) > 1),), g) for g in groups]


def needed_rows(ops, h, scale, ky0, ky1):
    """Rows [lo, hi) of every tensor that the kept output rows [ky0, ky1) depend on, each in its own resolution: walked
    back from the output through every consumer (a 3x3 convolution widens by one row on each side, clipped to the tile,
    beyond which it reads zero padding)."""
    need = {'out': (scale * ky0, scale * ky1)}
    for _, out, ins in reversed(ops):
        lo, hi = need[out]
        for t, how in ins:
            H = h * resolution(t, scale)
            if how == 'pw':
                a, b = lo, hi
            elif how == 'conv':
                a, b = max(lo - 1, 0), min(hi + 1, H)
            else:                                           # row y of the x2 grid reads source row y // 2
                a, b = max(lo - 1, 0) // 2, (min(hi + 1, 2 * H) + 1) // 2
            need[t] = (min(need[t][0], a), max(need[t][1], b)) if t in need else (a, b)
    return need


# ------------------------------------------------------------------------------------------------
# the workspace plan: where the forward keeps each tensor (csrc/k4_sr.cu, DESIGN.md section 3.4)
# ------------------------------------------------------------------------------------------------
def buffer_spec(scale):
    f16, f32 = torch.float16, torch.float32
    spec = {'in16': (f16, 32, 1), 'cond32': (f32, 32, 1), 'cond16': (f16, 32, 1), 'feat': (f32, 64, 1),
            'trunk_a': (f32, 64, 1), 'trunk_b': (f32, 64, 1), 'cat': (f16, 192, 1), 'cat2': (f16, 192, 1),
            'sbody': (f16, 64, 1), 'bf': (f16, 64, 1), 'hr': (f16, 64, scale)}
    if scale == 4:
        spec.update(up1=(f16, 64, 2), up2=(f16, 64, 4))
    return spec


def slots_of(t, fused):
    """(buffer, c0, c1) of each place tensor t is stored.  The dense blocks' concatenations share one buffer, or with SFT
    fused alternate between cat and cat2 (a conv5 writes the next block's xc0 while this block's is still read); a dense
    block's output goes to trunk B and an RRDB's output to trunk A, which conv_first initialises with feat."""
    if t == 'x':
        return [('in16', 0, 32)]
    if t == 'cond':
        return [('cond32', 0, 32)] + ([('cond16', 0, 32)] if fused else [])
    if t == 'feat':
        return [('feat', 0, 64), ('trunk_a', 0, 64)]
    if t in ('sbody', 'bf', 'up1', 'up2', 'hr'):
        return [(t, 0, 64)]
    name, r = t.split('.', 1)
    if name == 'rrdb':
        return [('trunk_a', 0, 64)]
    if name == 'y':
        return [('trunk_b', 0, 64)]
    i, j = (int(v) for v in r.split('.'))
    cat = 'cat2' if fused and (3 * i + j) & 1 else 'cat'
    c0 = {'xc0': 0, 'x1': 64, 'x2': 96, 'x3': 128, 'x4': 160, 'xc1': 160}[name]
    return [(cat, c0, c0 + (64 if name == 'xc0' else 32))]


class Workspace:
    """Typed [rows, cols, channels] views of a workspace (uint8 tensor) in the layout the library reports."""

    def __init__(self, layout, h, w, scale):
        self.spec, self.h, self.w = buffer_spec(scale), h, w
        self.off = {k: getattr(layout, k) for k in self.spec}
        assert len(set(self.off.values())) == len(self.off) and max(self.off.values()) < layout.total

    def view(self, ws, name):
        dt, cs, r = self.spec[name]
        esz = torch.finfo(dt).bits // 8
        n = r * self.h * r * self.w * cs * esz
        return ws[self.off[name]:self.off[name] + n].view(dt).view(r * self.h, r * self.w, cs)

    def byte_view(self, ws, name):
        dt, cs, r = self.spec[name]
        esz = torch.finfo(dt).bits // 8
        n = r * self.h * r * self.w * cs * esz
        return ws[self.off[name]:self.off[name] + n].view(r * self.h, r * self.w, cs * esz), esz


# ------------------------------------------------------------------------------------------------
# the prefix runs
# ------------------------------------------------------------------------------------------------
MAX_STEPS = 512


def forward_upto(net, x, c, keep, frame, out, ws, stop_after):
    """Poison the workspace and the output frame (out: a window of it), run the forward's first `stop_after` steps,
    synchronise.  Returns the step descriptors and the workspace layout."""
    h, w = x.shape[2], x.shape[3]
    ws.fill_(0xFF)
    frame.view(torch.uint8).fill_(0xFF)
    steps = (_lib.SrStep * MAX_STEPS)()
    n = C.c_int32(-1)
    lay = _lib.SrWsLayout()
    st = _lib.lib.k4_testing_srnet_forward_upto(net._get_net().ptr, x.data_ptr(), c.data_ptr(), h, w, *keep, out.data_ptr(),
                                                out.stride(0), out.stride(1), ws.data_ptr(), ws.numel(), stop_after, steps,
                                                MAX_STEPS, C.byref(n), C.byref(lay),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0, f'k4_testing_srnet_forward_upto -> {st} ({_lib.lib.k4_status_string(st).decode()})'
    torch.cuda.synchronize()
    assert 0 < n.value <= min(stop_after, MAX_STEPS)
    return [(_lib.SR_STEP_KINDS[s.kind], s.block, s.dense, s.conv, s.fused) for s in steps[:n.value]], lay


# ------------------------------------------------------------------------------------------------
# float64 layers with their element bounds
# ------------------------------------------------------------------------------------------------
def lrelu32(v):
    """LeakyReLU 0.2 as the epilogues apply it: one fp32 multiply by 0.2f."""
    v32 = v.float()
    return torch.where(v32 > 0, v32, v32 * torch.tensor(0.2, dtype=torch.float32)).double()


def conv_layer(mod, a, up):
    """a: fp64 [H, W, cin] operand.  Returns the fp64 output [OH, OW, cout] and its bound 2^-16 sum |a||w| + the
    sub-pixel weight allowance of conv_ref + a few fp32 roundings."""
    v, S, T = conv_ref(a.permute(2, 0, 1)[None], mod.weight.detach(), mod.bias.detach(), up, False)
    v, S, T = v.permute(1, 2, 0), S.permute(1, 2, 0), T.permute(1, 2, 0)
    return v, 2.0 ** -16 * S + T + FP32_EPS * v.abs()


def sft_weights(layer):
    return [t.detach().reshape(t.shape[0], -1) if t.dim() > 1 else t.detach() for cv in layer.convs()
            for t in (cv.weight, cv.bias)]


def sft_apply(layer, x, e_x, cond, fused):
    """y = x * (scale + 1) + shift of an SFT layer on x [H, W, cout] with bound e_x, and y's bound (test_sft_epilogues /
    test_sft_pass_meets_its_element_bound): the fused epilogues and the mma pass read the condition as fp16, the fp32
    pass (K4_SFT_FP32) as fp32."""
    H, W, n = x.shape
    p = sft_weights(layer)
    if fused:
        sc, e_sc, sh, e_sh = sft_ref(p, cond['cond16'].reshape(H * W, 32))
    elif 'K4_SFT_FP32' in os.environ:
        sc, e_sc, sh, e_sh = sft_ref32(p, cond['cond32'].reshape(H * W, 32))
    else:
        sc, e_sc, sh, e_sh = sft_ref(p, cond['cond32'].reshape(H * W, 32).clamp(-FP16_MAX, FP16_MAX).half())
    sc, e_sc, sh, e_sh = (t.view(H, W, n) for t in (sc, e_sc, sh, e_sh))
    y = x * sc + sh
    return y, e_x * sc.abs() + x.abs() * e_sc + e_sh + FP32_EPS * (y.abs() + (x * sc).abs())


def nets_layer(net, kind, i, j, c):
    if kind == 'conv_first':
        return net.conv_first
    if kind == 'rdb_conv':
        return getattr(getattr(net.body[i], f'rdb{j + 1}'), f'conv{c + 1}')
    if kind in ('sft0', 'sft1'):
        return getattr(getattr(net.body[i], f'rdb{j + 1}'), kind)
    if kind == 'sft_rrdb':
        return net.body[i].sft0
    if kind == 'sft_body':
        return net.sftbody
    return {'conv_body': net.conv_body, 'up1': getattr(net, 'conv_up1', None), 'up2': getattr(net, 'conv_up2', None),
            'hr': net.conv_hr, 'last': net.conv_last}[kind]


def condnet_check(net, cin, ws_prev, ws_cur, W_, rows, fused):
    kernel = FP32 if os.environ.get('K4_CONDNET_FP32', '0')[:1] == '1' else MMA
    p = [t.detach() for k in (0, 2, 4, 6) for t in (net.CondNet[k].weight, net.CondNet[k].bias)]
    if cin.shape[0] == 1:
        ref, E, _ = condnet_ref_depth(p, cin[0], kernel)
    else:
        ref, E, _ = condnet_ref_wide(p, cin, kernel)
    h, w = cin.shape[1:]
    got = W_.view(ws_cur, 'cond32')
    out = [('cond32', got[rows[0]:rows[1]].double(), ref.view(h, w, 32)[rows[0]:rows[1]], E.view(h, w, 32)[rows[0]:rows[1]])]
    if fused:       # cond16: the saturated fp16 rounding of the kernel's own cond32, bit for bit
        c16 = W_.view(ws_cur, 'cond16')[rows[0]:rows[1]]
        want = got[rows[0]:rows[1]].clamp(-FP16_MAX, FP16_MAX).half()
        assert torch.equal(c16.view(torch.int16), want.view(torch.int16)), 'cond16 is not the fp16 rounding of cond32'
    return out


def step_references(net, group, val, cond, fused):
    """fp64 value and bound of every tensor the step's layers produce, from the operands `val(t)` of the previous
    snapshot: (tensor, ref, bound, stored in fp16)."""
    res, prev = [], None
    for (kind, i, j, c), out, ins in group:
        if kind.startswith('sft'):
            x, e_x = prev if prev is not None else (val(ins[0][0]), 0.0)
            y, e_y = sft_apply(nets_layer(net, kind, i, j, c), x, e_x, cond, fused)
            if kind == 'sft_rrdb':                          # out * 0.2 + x_in
                r = val(ins[2][0])
                u = y * RES_SCALE + r
                y, e_y = u, RES_SCALE * e_y + FP32_EPS * (u.abs() + r.abs() + (y * RES_SCALE).abs())
        else:
            mod = nets_layer(net, kind, i, j, c)
            srcs = [t for t, how in ins if how != 'pw']
            a = torch.cat([val(t) for t in srcs], 2)
            if kind == 'conv_first':
                a = a[:, :, :3]
            y, e_y = conv_layer(mod, a, ins[0][1] == 'up')
            if kind == 'rdb_conv' and c == 4:              # x5 * 0.2 + x
                r = val(ins[-1][0])
                t_ = y * RES_SCALE + r
                y, e_y = t_, RES_SCALE * e_y + FP32_EPS * (t_.abs() + r.abs())
            elif kind == 'conv_body':                       # conv_body(...) + feat
                r = val('feat')
                t_ = y + r
                y, e_y = t_, e_y + FP32_EPS * (t_.abs() + r.abs())
            elif kind in ('rdb_conv', 'up1', 'up2', 'hr'):
                y = lrelu32(y)
        res.append((out, y, e_y))
        prev = (y, e_y)
    return res


# ------------------------------------------------------------------------------------------------
# one case: every step of one forward
# ------------------------------------------------------------------------------------------------
VARIANTS = {'x4': (4, 1), 'x4_pretrained': (4, 1), 'x1': (1, 1), 'cond63': (4, 63), 'cond64': (4, 64)}
_NETS = {}


def make_net(variant):
    if variant not in _NETS:
        scale, nc = VARIANTS[variant]
        if variant == 'x4_pretrained':
            from helpers import pretrained_sr_state_dict
            sd = pretrained_sr_state_dict()
            if sd is None:
                pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing')
        elif scale == 1:
            sd = x1_state_dict(seed=3)
        else:
            sd = sftnet.random_state_dict(seed=3, num_cond=nc)
        n = k4nerf.SFTNet(3, scale, 64, NUM_BLOCK, 32, nc)
        n.load_state_dict(sd)
        _NETS[variant] = n.cuda()
    return _NETS[variant]


def make_inputs(variant, h, w, seed=7):
    _, nc = VARIANTS[variant]
    g = torch.Generator().manual_seed(seed + h * 131 + w)
    x = torch.rand(1, 3, h, w, generator=g) * 1.2 - 0.1
    c = torch.rand(1, 1, h, w, generator=g) if nc == 1 else frame_condition(nc, h, w, seed)[None]
    return x.cuda().contiguous(), c.cuda().float().contiguous()


def check_elements(label, got, ref, bound, worst):
    got = got.double()
    if not bool(torch.isfinite(got).all()):
        idx = [int(v) for v in torch.nonzero(~torch.isfinite(got))[0]]
        raise AssertionError(f'{label}: {int((~torch.isfinite(got)).sum())} non-finite elements in rows it must produce, '
                             f'first at [y, x, c] = {idx}')
    d = (got - ref).abs()
    bad = d > bound
    if bool(bad.any()):
        idx = [int(v) for v in torch.nonzero(bad)[0]]
        raise AssertionError(f'{label}: {int(bad.sum())} of {d.numel()} elements over the bound, first at [y, x, c] = {idx}: '
                             f'{got[tuple(idx)].item()} vs {ref[tuple(idx)].item()} (bound {bound[tuple(idx)].item():.3g})')
    r = (d / bound.clamp_min(1e-300)).max().item() if d.numel() else 0.0
    worst[0] = max(worst[0], r)


def chain_case(variant, h, w, keep=None, fused=None):
    """Every step of one forward of `variant` on an h x w tile (keep: the LR block (y0, y1, x0, x1) kept, default the
    whole tile).  fused None: what the environment selects.  Returns {layer kind: largest error / bound}."""
    net = make_net(variant)
    scale, nc = VARIANTS[variant]
    if fused is None:
        fused = os.environ.get('K4_SR_FUSE_SFT', '1')[:1] != '0' and os.environ.get('K4_CONV_NO_TMA', '0')[:1] != '1'
    ky0, ky1, kx0, kx1 = keep if keep is not None else (0, h, 0, w)
    x, c = make_inputs(variant, h, w)
    ws = torch.empty(int(_lib.lib.k4_srnet_workspace_bytes(net._get_net().ptr, h, w)), dtype=torch.uint8, device=x.device)
    frame = torch.empty(3, scale * h + 3, scale * w + 5, device=x.device)     # the kept block lands at (1, 2) of it
    oy, ox = scale * ky0 + 1, scale * kx0 + 2
    out = frame[:, oy:oy + scale * (ky1 - ky0), ox:ox + scale * (kx1 - kx0)]
    ops = reference_ops(NUM_BLOCK, scale)
    plan = steps_of(ops, fused)
    need = needed_rows(ops, h, scale, ky0, ky1)
    descs, lay = forward_upto(net, x, c, (ky0, ky1, kx0, kx1), frame, out, ws, 10 ** 6)
    assert descs == [d for d, _ in plan], 'the launch sequence is not the reference structure'
    W_ = Workspace(lay, h, w, scale)
    consumers = {}
    for si, (_, g) in enumerate(plan):
        for _, _, ins in g:
            for t, _ in ins:
                consumers.setdefault(t, set()).add(si)
    where = {}
    worst = {}
    prev_ws, prev_frame = torch.full_like(ws, 0xFF), torch.full_like(frame.view(torch.uint8), 0xFF)
    for k, (desc, group) in enumerate(plan, start=1):
        got_descs, _ = forward_upto(net, x, c, (ky0, ky1, kx0, kx1), frame, out, ws, k)
        assert got_descs == descs[:k]
        cur_ws, cur_frame = ws.clone(), frame.view(torch.uint8).clone()
        kind = desc[0]
        label = f'{variant} {h}x{w} {"fused" if fused else "unfused"} step {k} {desc}'
        wk = worst.setdefault(kind + ('+sft' if desc[4] else ''), [0.0])
        # what the step writes: every tensor of its layers that a later step reads, the output, and an RRDB's output
        # (the trunk, kept in trunk A even where only the fused sftbody reads it)
        stored = [t for _, t, _ in group
                  if t == 'out' or t.startswith('rrdb.') or any(s != k - 1 for s in consumers.get(t, ()))]
        declared = [s for t in stored if t != 'out' for s in slots_of(t, fused)]
        # and on which rows: the rows the later layers need; the input conversion covers the tile, and CondNet runs once
        # for every SFT layer, so its row extent is not constrained
        declared_rows = [(s, (0, None) if t in ('x', 'cond') else need[t])
                         for t in stored if t != 'out' for s in slots_of(t, fused)]

        def val(t):
            assert where.get(t), f'{label}: operand {t} is not in the workspace any more'
            b, c0, c1 = where[t][0]
            return W_.view(prev_ws, b)[:, :, c0:c1].double()

        if kind == 'input':
            v = W_.view(cur_ws, 'in16')
            assert torch.equal(v[:, :, :3], x[0].permute(1, 2, 0).half()) and bool((v[:, :, 3:] == 0).all()), label
        elif kind == 'condnet':
            lo, hi = need['cond']
            for name, g_, r_, b_ in condnet_check(net, c[0], prev_ws, cur_ws, W_, (lo, hi), fused):
                check_elements(f'{label} {name}', g_, r_, b_, wk)
        else:
            cond = {k_: W_.view(prev_ws, k_)[:, :, :32].double() for k_ in ('cond32', 'cond16')}
            for t, ref, bound in step_references(net, group, val, cond, desc[4] == 1):
                if t not in stored:
                    continue
                lo, hi = need[t]
                if t == 'out':
                    got = out.permute(1, 2, 0)
                    ref, bound = ref[lo:hi, scale * kx0:scale * kx1], bound[lo:hi, scale * kx0:scale * kx1]
                    check_elements(f'{label} out', got, ref, bound, wk)
                    continue
                for (b, c0, c1) in slots_of(t, fused):
                    got = W_.view(cur_ws, b)[lo:hi, :, c0:c1]
                    bd = bound[lo:hi]
                    if W_.spec[b][0] == torch.float16:
                        bd = bd + 0.5 * ulp16(ref[lo:hi].abs() + bd)
                    check_elements(f'{label} {t} in {b}[{c0}:{c1}]', got, ref[lo:hi], bd, wk)
        # nothing outside the declared output (buffer, channels, rows) changed; the frame only inside the kept block, by
        # the last step
        changed = prev_ws != cur_ws
        for (b, c0, c1), (lo, hi) in declared_rows:
            bv, esz = W_.byte_view(changed, b)
            bv[lo:hi, :, c0 * esz:c1 * esz] = False
        if bool(changed.any()):
            pos = int(torch.nonzero(changed)[0])
            owner = max((o, n_) for n_, o in W_.off.items() if o <= pos)
            bv, esz = W_.byte_view(changed, owner[1])
            at = [int(v) for v in torch.nonzero(bv)[0]]
            raise AssertionError(f'{label}: wrote outside its declared output {declared_rows}: {owner[1]} at [y, x, byte] = {at}')
        fchanged = (prev_frame != cur_frame).view(frame.shape[0], frame.shape[1], frame.shape[2], 4).any(-1)
        if kind == 'last':
            fchanged[:, oy:oy + out.shape[1], ox:ox + out.shape[2]] = False
        assert not bool(fchanged.any()), f'{label}: wrote into the frame outside the kept block'
        for t in list(where):                              # slots overwritten by this step no longer hold their tensor
            where[t] = [s for s in where[t] if not any(s[0] == d[0] and s[1] < d[2] and d[1] < s[2] for d in declared)]
        for t in stored:
            if t != 'out':
                where[t] = slots_of(t, fused)
        prev_ws, prev_frame = cur_ws, cur_frame
    # the last prefix run is the whole forward: the same frame as net(x, c), bit for bit
    full = net(x, c)[0, :, scale * ky0:scale * ky1, scale * kx0:scale * kx1]
    assert torch.equal(out, full), f'{variant} {h}x{w}: the stepped forward differs from net(x, c)'
    ratios = {k_: v[0] for k_, v in worst.items()}
    print(f'chain {variant} {h}x{w} keep {(ky0, ky1, kx0, kx1)} {"fused" if fused else "unfused"}: largest |y - ref| / bound '
          + ', '.join(f'{k_} {v:.3g}' for k_, v in ratios.items()))
    return ratios


SIZES = [(19, 13), (1, 7), (96, 128)]


@pytest.mark.parametrize('fused', (True, False), ids=('fused', 'unfused'))
@pytest.mark.parametrize('hw', SIZES, ids=lambda s: f'{s[0]}x{s[1]}')
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_every_layer_of_the_forward_meets_its_bound_in_place(variant, hw, fused, monkeypatch, cuda_device):
    """The whole tile kept: every layer of the real forward, on the operands the forward left in the workspace, within
    its element bound on every row, and nothing else changed.  19x13 is ragged against every tile shape, 1x7 a single
    row, 96x128 makes every convolution's ring wrap.  K4_SR_FUSE_SFT is read per call."""
    monkeypatch.setenv('K4_SR_FUSE_SFT', '1' if fused else '0')
    if fused and os.environ.get('K4_CONV_NO_TMA', '0')[:1] == '1':
        pytest.skip('K4_CONV_NO_TMA=1 runs every SFT layer as its own pass')
    chain_case(variant, *hw, fused=fused)


@pytest.mark.parametrize('fused', (True, False), ids=('fused', 'unfused'))
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_forward_roi_reads_only_rows_it_computed(variant, fused, monkeypatch, cuda_device):
    """forward_roi with a kept block strictly inside a 96x128 tile: each layer is checked on the rows the layers behind
    it still need, which narrow from the whole tile (the trunk's first blocks) to the kept block plus its tail's context.
    The workspace starts as NaN, so a layer that reads a row no layer computed in this call fails its check."""
    monkeypatch.setenv('K4_SR_FUSE_SFT', '1' if fused else '0')
    if fused and os.environ.get('K4_CONV_NO_TMA', '0')[:1] == '1':
        pytest.skip('K4_CONV_NO_TMA=1 runs every SFT layer as its own pass')
    chain_case(variant, 96, 128, keep=(41, 53, 30, 91), fused=fused)


# ------------------------------------------------------------------------------------------------
# the decoder's per-process switches, in child interpreters
# ------------------------------------------------------------------------------------------------
_CHILD = r'''
import sys
sys.path[:0] = [sys.argv[1], sys.argv[1] + '/4k-nerf_b200', sys.argv[1] + '/tests']
import test_gpu_sftnet_chain as T
T.chain_case('x4', 19, 13)
'''
SWITCHES = ('K4_CONV_K64', 'K4_CONV_NO_TMA', 'K4_SR_PDL', 'K4_SFT_FP32', 'K4_SR_FUSE_SFT', 'K4_CONDNET_FP32')


@pytest.mark.parametrize('env', [{'K4_CONV_K64': '0'}, {'K4_CONV_NO_TMA': '1'}, {'K4_CONDNET_FP32': '1'}],
                         ids=lambda e: '-'.join(f'{k}={v}' for k, v in e.items()))
def test_every_layer_under_each_kernel_switch(env, tmp_path, cuda_device):
    """K4_CONV_K64=0 (every 64-channel layer on conv3x3_ws_kernel), K4_CONV_NO_TMA=1 (cp.async producers, SFT as its own
    passes) and K4_CONDNET_FP32=1 (the fp32 CondNet kernel) change the kernel of whole sets of layers and are latched at
    a process's first decoder call: the 19x13 x4 case runs in a child interpreter for each."""
    base = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, '-c', _CHILD, ROOT], env=dict(base, **env), cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


# ------------------------------------------------------------------------------------------------
# tile_process: the reference's tiling, bit for bit
# ------------------------------------------------------------------------------------------------
TILE_GEOMS = [(150, 170, 64, 10), (40, 50, 64, 10), (128, 192, 64, 10), (40, 7, 16, 10)]
TILE_MODELS = ('x4', 'x1', 'cond64')


def tiled_by_the_plan(net, img, cond, tile_size, tile_pad):
    """The frame of lib/sr_esrnet.py:467-527 assembled here: net.forward on each padded tile of oracle.sftnet.tile_plan,
    the tile's un-padded block cropped out of its output."""
    s = net.scale
    _, _, H, W = img.shape
    frame = torch.full((1, 3, H * s, W * s), float('nan'), device=img.device)
    for (y0p, y1p, x0p, x1p, y0, y1, x0, x1, ty, tx) in sftnet.tile_plan(H, W, tile_size, tile_pad):
        t = net(img[:, :, y0p:y1p, x0p:x1p].contiguous(), cond[None, :, y0p:y1p, x0p:x1p].contiguous())
        frame[:, :, y0 * s:y1 * s, x0 * s:x1 * s] = t[:, :, ty * s:(ty + y1 - y0) * s, tx * s:(tx + x1 - x0) * s]
    return frame


@pytest.mark.parametrize('streams', (1, 2))
@pytest.mark.parametrize('geom', TILE_GEOMS, ids=lambda g: f'{g[0]}x{g[1]}-t{g[2]}-p{g[3]}')
@pytest.mark.parametrize('variant', TILE_MODELS)
def test_tile_process_is_the_reference_tiling_bit_for_bit(variant, geom, streams, cuda_device):
    """Ragged last tiles (150x170 at tile 64), a frame smaller than one tile, a tile size that divides the frame, a frame
    narrower than tile_pad; one and two streams."""
    H, W, ts, pad = geom
    net = make_net(variant)
    x, c = make_inputs(variant, H, W, seed=17)
    want = tiled_by_the_plan(net, x, c[0], ts, pad)
    got = net.tile_process(x, c[0], ts, pad, to_cpu=False, streams=streams)
    assert torch.equal(got, want)


@pytest.mark.parametrize('geom', TILE_GEOMS, ids=lambda g: f'{g[0]}x{g[1]}-t{g[2]}-p{g[3]}')
@pytest.mark.parametrize('variant', TILE_MODELS)
def test_tile_process_sharded_on_one_process_is_the_reference_tiling(variant, geom, cuda_device):
    H, W, ts, pad = geom
    net = make_net(variant)
    x, c = make_inputs(variant, H, W, seed=19)
    assert torch.equal(net.tile_process_sharded(x, c[0], ts, pad), tiled_by_the_plan(net, x, c[0], ts, pad))
