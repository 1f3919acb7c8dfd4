"""GPU: every VC-Decoder convolution kernel of csrc/k4_sr.cu, one layer at a time, against a float64 reference.

k4_testing_conv3x3 packs a layer with the packers k4_srnet_create uses (make_conv, make_conv_phases, make_conv_k64,
make_sft) and runs it through the decoder's dispatcher with a chosen kernel: conv3x3_ws_kernel with its TMA or its
cp.async producer, or conv3x3_k64_kernel.  The reference is F.conv2d in float64 on the GPU (after a nearest x2
upsampling for the up layers), followed by the epilogue written out in torch and, for the fused modes, the SFT MLPs
in float64.

(a) exact operands: torch.equal against the reference; (b) random operands: the precision contract of DESIGN.md,
element by element; (c) the fused SFT epilogues; (d) CondNet, both kernels (k4_testing_condnet); (e) the standalone
SFT pass, both kernels, in the decoder's four I/O forms (k4_testing_sft); (f) the fp16 saturation of the condition;
and, in child interpreters, the whole network under each of the decoder's A/B environment switches.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from k4nerf import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTO, WS_TMA, WS_CP, K64 = (_lib.K4_CONV_KERNEL_AUTO, _lib.K4_CONV_KERNEL_WS_TMA, _lib.K4_CONV_KERNEL_WS_CPASYNC,
                            _lib.K4_CONV_KERNEL_K64)
KNAME = {AUTO: 'auto', WS_TMA: 'ws_tma', WS_CP: 'ws_cpasync', K64: 'k64'}
OK, UNSUPPORTED = 0, -2
SENT16 = -7.0                    # sentinel of every destination: what a kernel must not write keeps it
SENT32 = -7.25
FP16_MAX = 65504.0


def npad_of(cout):
    return 16 if cout <= 16 else (32 if cout <= 32 else 64)


def cpad_of(cin):
    return (cin + 31) // 32 * 32


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------
# the C entry point
# ------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else t.data_ptr()


def _sft_ptrs(ts):
    return None if ts is None else C.cast((C.c_void_p * 8)(*[t.data_ptr() for t in ts]), C.POINTER(C.c_void_p))


def run_layer(w, b, src, kernel, *, src_c0=0, up=False, mode=0, lrelu=0.0, scale=1.0, scale2=1.0, rows=None,
              dst_h=None, dst_c0=0, dst_f=None, dst_f2=None, add_f=None, add_f2=None, dst_h2=None, dst2_c0=0,
              out=None, n_valid=0, crop=None, cond16=None, sft=None, sft2=None):
    """One k4_testing_conv3x3 call on the current stream.  src: fp16 [H, W, cstride]; dst_h / dst_h2: fp16 [.., .., cstride];
    dst_f / add_f: fp32 [pixels, 64]; out: fp32 view [c, y, x] of the crop window (unit stride along x).  Returns
    (status, kernel that ran)."""
    H, W, cs = src.shape
    a = _lib.ConvTestArgs()
    a.d_weight, a.d_bias, a.cout, a.cin = w.data_ptr(), b.data_ptr(), w.shape[0], w.shape[1]
    a.d_src, a.src_cstride, a.src_c0, a.H, a.W = src.data_ptr(), cs, src_c0, H, W
    a.upsample2x, a.mode, a.lrelu, a.scale, a.scale2 = int(up), mode, lrelu, scale, scale2
    a.y_lo, a.y_hi = rows if rows is not None else (0, H)
    a.d_dst_h, a.dst_cstride, a.dst_c0 = _ptr(dst_h), (dst_h.shape[-1] if dst_h is not None else 0), dst_c0
    a.d_dst_f, a.d_dst_f2, a.d_add_f, a.d_add_f2 = _ptr(dst_f), _ptr(dst_f2), _ptr(add_f), _ptr(add_f2)
    a.d_dst_h2, a.dst2_cstride, a.dst2_c0 = _ptr(dst_h2), (dst_h2.shape[-1] if dst_h2 is not None else 0), dst2_c0
    if out is not None:
        assert out.stride(2) == 1
        a.d_out_nchw, a.n_valid, a.out_plane_stride, a.out_row_stride = out.data_ptr(), n_valid, out.stride(0), out.stride(1)
        a.crop_y0, a.crop_y1, a.crop_x0, a.crop_x1 = crop
    a.d_cond16 = _ptr(cond16)
    a.h_sft, a.h_sft2 = _sft_ptrs(sft), _sft_ptrs(sft2)
    a.kernel = kernel
    used = C.c_int32(-9)
    st = _lib.lib.k4_testing_conv3x3(C.byref(a), C.byref(used), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return st, used.value


def expect_ran(st, used, kernel):
    assert st == OK, f'k4_testing_conv3x3 -> {st} ({_lib.lib.k4_status_string(st).decode()}) for kernel {KNAME[kernel]}'
    if kernel != AUTO:
        assert used == kernel, (KNAME[kernel], used)


# ------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------
# phase py of "nearest x2, then 3x3": source offset iy of the 2x2 footprint collects kernel rows R[py][iy]
_PHASE_ROWS = [[[1, 0, 0], [0, 1, 1]], [[1, 1, 0], [0, 0, 1]]]


def ulp16(x):
    """Spacing of the fp16 numbers around |x| (fp64 tensor; subnormal spacing below 2^-14)."""
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), (e.clamp_min(-13) - 11))


def tie_slack(x, e):
    """One fp16 ulp where x +- e round to different fp16 values (the kernel's value, within e of x, may round to the
    neighbour of the reference's fp16 rounding), else 0."""
    return torch.where((x + e).half() != (x - e).half(), ulp16(x.abs() + e), torch.zeros_like(x))


def conv_ref(a, w, b, up, exact):
    """a: fp64 [1, cin, H, W] (fp16 values), w fp32 [cout, cin, 3, 3].  Returns the fp64 output [cout, OH, OW], S = sum
    |a| |w16| over each output's products, and T, the allowance for the phase-combined weights of the sub-pixel form
    (0 for a direct convolution); (v, None, None) for exact operands, where the reference is the plain nearest upsampling
    followed by conv2d.  A layer's accumulation bound is 2^-16 S + T.

    T is sum |a| ulp16(w) over the combined weights whose fp32 sum may round to the neighbouring fp16 value of the
    fp64 sum's rounding.  It is a difference of one fp16 ulp in the operand itself, so it is not scaled by 2^-16 like
    the accumulation: conv_up2 of the num_cond 64 decoder (oracle.sftnet.random_state_dict(seed=3)) has such a weight,
    [11, 60] of tap (0, 0) of phase (1, 1), whose exact sum -0.0173568707 lies 1.9e-9 from an fp16 rounding boundary,
    and the kernel's weight is one ulp (1.5e-5) away from the reference's."""
    bd = b.double()
    if exact:
        x = F.interpolate(a, scale_factor=2, mode='nearest') if up else a
        return F.conv2d(x, w.double(), bd, padding=1)[0], None, None
    if not up:
        w16 = w.half().double()
        v = F.conv2d(a, w16, bd, padding=1)[0]
        return v, F.conv2d(a.abs(), w16.abs(), padding=1)[0], torch.zeros_like(v)
    # the sub-pixel form: each phase's combined weight formed in fp64 from the fp32 weights, rounded to fp16 once
    _, cin, H, W = a.shape
    ap = F.pad(a, (1, 1, 1, 1))
    R = torch.tensor(_PHASE_ROWS, dtype=torch.float64, device=a.device)
    y = torch.empty(w.shape[0], 2 * H, 2 * W, dtype=torch.float64, device=a.device)
    s, t = torch.empty_like(y), torch.empty_like(y)
    for py in (0, 1):
        for px in (0, 1):
            wp = torch.einsum('ik,jl,ockl->ocij', R[py], R[px], w.double())
            e = 2.0 ** -22 * torch.einsum('ik,jl,ockl->ocij', R[py], R[px], w.double().abs())
            wp16 = wp.half().double()
            win = ap[:, :, py:py + H + 1, px:px + W + 1]
            y[:, py::2, px::2] = F.conv2d(win, wp16, bd)[0]
            s[:, py::2, px::2] = F.conv2d(win.abs(), wp16.abs())[0]
            t[:, py::2, px::2] = F.conv2d(win.abs(), tie_slack(wp, e))[0]
    return y, s, t


def pad_channels(t, n):
    """[c, ...] -> [n, ...], zero channels appended (the npad outputs beyond cout)."""
    return torch.cat([t, t.new_zeros((n - t.shape[0],) + tuple(t.shape[1:]))]) if t.shape[0] < n else t


def hwc(t):
    """[c, h, w] -> [h*w, c]"""
    return t.permute(1, 2, 0).reshape(-1, t.shape[0])


# ------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------
def exact_operands(H, W, cs, cout, cin, seed, dev):
    """Activations k/16 (|k| <= 16), weights j/64 (|j| <= 8), biases on the 2^-10 grid: see test_exact_layers."""
    g = torch.Generator().manual_seed(seed)
    src = (torch.randint(-16, 17, (H, W, cs), generator=g) / 16.0).half()
    w = torch.randint(-8, 9, (cout, cin, 3, 3), generator=g) / 64.0
    b = torch.randint(-64, 65, (cout,), generator=g) / 1024.0
    return src.to(dev), w.to(dev), b.to(dev)


def random_operands(H, W, cs, cout, cin, seed, dev, weight=None):
    """Activations uniform in [-1, 2] (fp16), weights as the reference initialises its convolutions (Kaiming normal
    x 0.1) or given, biases N(0, 0.01^2)."""
    g = torch.Generator().manual_seed(seed)
    src = (torch.rand(H, W, cs, generator=g) * 3 - 1).half()
    if weight is None:
        weight = torch.randn(cout, cin, 3, 3, generator=g) * (math.sqrt(2.0 / (cin * 9)) * 0.1)
        bias = torch.randn(cout, generator=g) * 0.01
    else:
        weight, bias = weight
    return src.to(dev), weight.float().contiguous().to(dev), bias.float().contiguous().to(dev)


def trunk_operand(P, seed, dev, exact):
    """fp32 [P, 64] residual input: the 2^-12 grid within +-4 (exact sums) or uniform in [-1, 1]."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(-2 ** 14, 2 ** 14 + 1, (P, 64), generator=g) / 4096.0 if exact else torch.rand(P, 64, generator=g) * 2 - 1
    return t.to(dev)


# ------------------------------------------------------------------------------------------------
# one plain layer (modes 0-4): run, and return [(name, got, ref, bound or None)] plus the sentinel checks
# ------------------------------------------------------------------------------------------------
FP32_EPS = 2.0 ** -22            # a few fp32 roundings of the epilogue, relative to the magnitudes involved


def plain_layer(kernel, cout, cin, H, W, *, mode=0, lrelu=0.0, up=False, rows=None, operands='exact', seed=0,
                weight=None, dev='cuda'):
    s_ = 2 if up else 1
    OH, OW = H * s_, W * s_
    npad, cpad = npad_of(cout), cpad_of(cin)
    cs = cpad + 8                                   # the layer reads channels [8, 8 + cpad) of a wider buffer
    if operands == 'random':
        src, w, b = random_operands(H, W, cs, cout, cin, seed, dev, weight)
    else:
        src, w, b = exact_operands(H, W, cs, cout, cin, seed, dev)
    if operands == 'sat':
        # activations +-2^10 (one negative block), weights 7/64 or 8/64 with one sign per output channel, no bias: every
        # sum is an integer below 2^17 (exact), interior sums exceed 65504
        g = torch.Generator().manual_seed(seed)
        src = torch.full((H, W, cs), 1024.0)
        src[H // 2:H // 2 + 3, W // 4:W // 2] = -1024.0
        src = src.half().to(dev)
        sign = torch.where(torch.arange(cout) % 2 == 0, 1.0, -1.0).view(-1, 1, 1, 1)
        w = (torch.randint(7, 9, (cout, cin, 3, 3), generator=g) / 64.0 * sign).to(dev)
        b = torch.zeros_like(b)
    exact = operands != 'random'
    a = src[:, :, 8:8 + cin].permute(2, 0, 1)[None].double()
    v, S, T = conv_ref(a, w, b, up, exact)
    v, S, T = pad_channels(v, npad), (pad_channels(S, npad) if S is not None else None), (pad_channels(T, npad) if T is not None else None)
    ylo, yhi = rows if rows is not None else (0, H)
    rsel = slice(ylo * s_, yhi * s_)
    P = OH * OW
    bufs, checks = {}, []
    kw = dict(src_c0=8, up=up, mode=mode, lrelu=lrelu, rows=rows)
    errv = None if exact else 2.0 ** -16 * S + T + FP32_EPS * v.abs()

    def f16(name, ref, err):
        bound = None if exact else (err + 0.5 * ulp16(ref.abs() + err))[:, rsel]
        checks.append((name, bufs[name][rsel, :, 16:16 + npad].permute(2, 0, 1), ref[:, rsel].float().clamp(-FP16_MAX, FP16_MAX).half()
                       if exact else ref[:, rsel], bound))

    def f32(name, ref, err):
        checks.append((name, bufs[name].view(OH, OW, 64)[rsel, :, :npad].permute(2, 0, 1), ref[:, rsel].float() if exact else ref[:, rsel],
                       None if exact else err[:, rsel]))

    if mode == 0:
        bufs['dst_h'] = torch.full((OH, OW, npad + 24), SENT16, dtype=torch.float16, device=dev)
        kw.update(dst_h=bufs['dst_h'], dst_c0=16)
        ref = v
        if lrelu > 0:                               # the kernel's single fp32 multiply
            v32 = v.float()
            ref = torch.where(v32 > 0, v32, v32 * torch.tensor(lrelu, dtype=torch.float32)).double()
        f16('dst_h', ref, errv)
    elif mode in (1, 2):
        add = trunk_operand(P, seed + 1, dev, exact)
        kw['add_f'] = add
        addr = add.view(OH, OW, 64).permute(2, 0, 1)[:npad].double()
        if mode == 1:
            bufs['dst_f'] = torch.full((P, 64), SENT32, device=dev)
            kw.update(dst_f=bufs['dst_f'], scale=0.25)
            ref = v * 0.25 + addr
            f32('dst_f', ref, None if exact else 0.25 * errv + FP32_EPS * (addr.abs() + ref.abs()))
        else:
            bufs['dst_h'] = torch.full((OH, OW, npad + 24), SENT16, dtype=torch.float16, device=dev)
            kw.update(dst_h=bufs['dst_h'], dst_c0=16)
            ref = v + addr
            f16('dst_h', ref, None if exact else errv + FP32_EPS * (addr.abs() + ref.abs()))
    elif mode == 3:
        for k in ('dst_f', 'dst_f2'):
            bufs[k] = torch.full((P, 64), SENT32, device=dev)
        kw.update(dst_f=bufs['dst_f'], dst_f2=bufs['dst_f2'])
        f32('dst_f', v, errv)
        f32('dst_f2', v, errv)
    elif mode == 4:                                 # conv_last: n_valid planes into a cropped window of a strided frame
        frame = torch.full((4, OH + 5, OW + 9), SENT32, device=dev)
        cy0, cy1, cx0, cx1 = min(1, OH - 1), OH, min(2, OW - 1), max(min(2, OW - 1) + 1, OW - 1)
        win = frame[:3, 3:3 + cy1 - cy0, 4:4 + cx1 - cx0]
        bufs['frame'] = frame
        kw.update(out=win, n_valid=3, crop=(cy0, cy1, cx0, cx1))
        ry0, ry1 = max(cy0, ylo * s_), min(cy1, yhi * s_)
        got = win[:, ry0 - cy0:max(ry0, ry1) - cy0]
        sub = (slice(0, 3), slice(ry0, max(ry0, ry1)), slice(cx0, cx1))
        checks.append(('out_nchw', got, v[sub].float() if exact else v[sub], None if exact else errv[sub]))
        mask = torch.ones_like(frame, dtype=torch.bool)
        mask[:3, 3 + ry0 - cy0:3 + max(ry0, ry1) - cy0, 4:4 + cx1 - cx0] = False
        bufs['frame_mask'] = mask
    st, used = run_layer(w, b, src, kernel, **kw)
    return st, used, bufs, checks, (rsel, npad)


def assert_untouched(bufs, rsel, npad, OH):
    """Everything a layer must not write still holds the sentinel, bit for bit."""
    for k, t in bufs.items():
        if k == 'dst_h':
            m = torch.ones_like(t, dtype=torch.bool)
            m[rsel, :, 16:16 + npad] = False
            assert bool((t[m] == SENT16).all()), f'{k}: wrote outside rows/channels'
        elif k in ('dst_f', 'dst_f2'):
            m = torch.ones_like(t, dtype=torch.bool)
            m.view(OH, -1, 64)[rsel, :, :npad] = False
            assert bool((t[m] == SENT32).all()), f'{k}: wrote outside rows/channels'
        elif k == 'frame':
            assert bool((t[bufs['frame_mask']] == SENT32).all()), 'out_nchw: wrote outside the crop window / n_valid planes'


def check_exact(checks):
    for name, got, ref, _ in checks:
        if not torch.equal(got, ref):
            d = (got.double() - ref.double()).abs()
            idx = [int(i) for i in torch.nonzero(d)[0]]
            raise AssertionError(f'{name}: {int((d > 0).sum())} of {d.numel()} elements differ, first at [c, y, x] = {idx}: '
                                 f'{got[tuple(idx)].item()} vs {ref[tuple(idx)].item()}')
        assert torch.isfinite(got.float()).all(), name


def check_bound(checks, label):
    worst = 0.0
    for name, got, ref, bound in checks:
        assert torch.isfinite(got.float()).all(), name
        r = (got.double() - ref).abs() / bound
        worst = max(worst, r.max().item())
        if not bool((r <= 1.0).all()):
            idx = [int(i) for i in torch.nonzero(r > 1.0)[0]]
            raise AssertionError(f'{name}: {int((r > 1).sum())} elements over the bound, max ratio {r.max().item():.3g}; '
                                 f'first at {idx}: {got[tuple(idx)].item()} vs {ref[tuple(idx)].item()} (bound {bound[tuple(idx)].item():.3g})')
    print(f'{label}: largest |y - ref| / bound = {worst:.3g}')
    return worst


# ------------------------------------------------------------------------------------------------
# (a) exact operands
# ------------------------------------------------------------------------------------------------
# (kernel, cout, cin, up): the ws kernel at every output width and every input width of the decoder, directly and, on the
# decoder's up layers (64 -> 64), in the sub-pixel x2 form; the k64 kernel at its two widths and on the up layers
KERNEL_CFGS = ([(k, n, ci, False) for k in (WS_TMA, WS_CP) for n in (16, 32, 64) for ci in (32, 64, 96, 128, 160, 192)]
               + [(K64, 16, 64, False), (K64, 64, 64, False)]
               + [(k, 64, 64, True) for k in (WS_TMA, WS_CP, K64)])
KERNELS_64 = (WS_TMA, WS_CP, K64)           # the three kernels of a 64 -> 64 layer


def _cfg_id(c):
    k, n, ci, up = c
    return f'{KNAME[k]}-n{n}-cin{ci}' + ('-up2x' if up else '')


def run_exact(kernel, cout, cin, H, W, **kw):
    st, used, bufs, checks, (rsel, npad) = plain_layer(kernel, cout, cin, H, W, **kw)
    expect_ran(st, used, kernel)
    torch.cuda.synchronize()
    check_exact(checks)
    assert_untouched(bufs, rsel, npad, (2 if kw.get('up') else 1) * H)
    return bufs, checks


@pytest.mark.parametrize('cfg', KERNEL_CFGS, ids=_cfg_id)
def test_exact_layers(cfg, cuda_device):
    """Operands on coarse grids make every product and every partial sum exact in fp32: activations k/16 (|k| <= 16),
    weights j/64 (|j| <= 8), biases on the 2^-10 grid.  All products then lie on the 2^-10 grid and |sum| <= 1728 * 1/8
    < 2^8 even at cin = 192 -- 18 significant bits, 6 below what the tensor cores' alignment / truncation of the fp32
    accumulation could cost -- and the phase-combined weights of the sub-pixel layers (sums of <= 4 weights) are exact
    in fp16 too.  So every fp32 output must EQUAL the fp64 result and every fp16 output must equal its correctly rounded
    (saturated) value: any wrong tap, phase, channel block, swizzle row, halo row, tile edge or stride shows up as a
    nonzero difference, not as a few tenths of a dB."""
    k, n, ci, up = cfg
    run_exact(k, n, ci, 17, 33, mode=0, lrelu=0.2, up=up, seed=ci + n)


MODES = [(0, 0.0), (0, 0.2), (1, 0.0), (2, 0.0), (3, 0.0), (4, 0.0)]


@pytest.mark.parametrize('kernel', KERNELS_64, ids=KNAME.get)
@pytest.mark.parametrize('mode_lrelu', MODES, ids=lambda m: f'mode{m[0]}' + ('-lrelu' if m[1] else ''))
def test_exact_epilogue_modes(kernel, mode_lrelu, cuda_device):
    """Every plain epilogue on a 64 -> 64 layer (mode 4: conv_last, 64 -> 3 padded to 16 outputs, three planes into a
    cropped window of a strided frame).  k64 runs only modes 0, 2 and 4 and must refuse the others."""
    mode, lrelu = mode_lrelu
    cout = 3 if mode == 4 else 64
    if kernel == K64 and mode in (1, 3):
        st, used, *_ = plain_layer(kernel, cout, 64, 17, 33, mode=mode, lrelu=lrelu)
        assert (st, used) == (UNSUPPORTED, -1)
        return
    run_exact(kernel, cout, 64, 17, 33, mode=mode, lrelu=lrelu, seed=mode)


SHAPES_W = (1, 7, 23, 24, 25, 31, 32, 33, 97)
SHAPES_H = (1, 15, 16, 17)


@pytest.mark.parametrize('kernel', KERNELS_64, ids=KNAME.get)
@pytest.mark.parametrize('H', SHAPES_H)
@pytest.mark.parametrize('W', SHAPES_W)
def test_exact_shapes(kernel, H, W, cuda_device):
    """Widths around the 24- (k64) and 32-pixel (ws) tile widths, heights around the 16-row tile height, down to 1x1."""
    run_exact(kernel, 64, 64, H, W, mode=0, lrelu=0.2, seed=H * 100 + W)


RING_CFGS = [(WS_TMA, 64, 64), (WS_CP, 64, 64), (WS_TMA, 32, 160), (WS_CP, 16, 96), (K64, 64, 64), (K64, 16, 64)]


@pytest.mark.parametrize('kernel,cout,cin', RING_CFGS, ids=[f'{KNAME[k]}-n{n}-cin{ci}' for k, n, ci in RING_CFGS])
def test_exact_many_tiles_wrap_every_ring(kernel, cout, cin, cuda_device):
    """More than 3 x SM-count tiles: every persistent CTA wraps its shared-memory ring (k64: 2 stages at N = 64) and
    flips the mbarrier phase parity several times."""
    tx = 24 if kernel == K64 else 32
    W = 40 * tx - 5
    H = 16 * (3 * sm_count() // 40 + 2) - 3
    assert ((W + tx - 1) // tx) * ((H + 15) // 16) > 3 * sm_count()
    run_exact(kernel, cout, cin, H, W, mode=0, lrelu=0.2, seed=7)


@pytest.mark.parametrize('kernel,up', [(WS_TMA, False), (WS_CP, False), (K64, False), (WS_TMA, True), (K64, True)],
                         ids=lambda v: KNAME.get(v) if isinstance(v, int) and not isinstance(v, bool) else ('up2x' if v else 'direct'))
@pytest.mark.parametrize('rows', [(5, 6), (3, 37), (16, 33)], ids=lambda r: f'rows{r[0]}-{r[1]}')
def test_exact_row_windows(kernel, up, rows, cuda_device):
    """A launch computing rows [y_lo, y_hi) strictly inside the image: its halo reads the real neighbouring rows (not
    padding) and the rows outside the window keep their sentinel."""
    run_exact(kernel, 64, 64, 40, 29, mode=0, lrelu=0.2, up=up, rows=rows, seed=rows[0])


@pytest.mark.parametrize('kernel', (WS_TMA, WS_CP), ids=KNAME.get)
@pytest.mark.parametrize('c', range(4))
def test_exact_dense_block_concat_in_place(kernel, c, cuda_device):
    """conv{c+1} of a dense block: reads channels [0, 64 + 32c) of the 192-channel buffer and writes its 32 growth
    channels at 64 + 32c INTO THE SAME BUFFER; every other channel stays byte-identical."""
    H, W, cin = 19, 45, 64 + 32 * c
    src, w, b = exact_operands(H, W, 192, 32, cin, 40 + c, 'cuda')
    before = src.clone()
    a = src[:, :, :cin].permute(2, 0, 1)[None].double()
    v, *_ = conv_ref(a, w, b, False, True)
    v32 = v.float()
    ref = torch.where(v32 > 0, v32, v32 * torch.tensor(0.2, dtype=torch.float32)).half()
    st, used = run_layer(w, b, src, kernel, mode=0, lrelu=0.2, dst_h=src, dst_c0=64 + 32 * c)
    expect_ran(st, used, kernel)
    torch.cuda.synchronize()
    assert torch.equal(src[:, :, 64 + 32 * c:96 + 32 * c].permute(2, 0, 1), ref)
    keep = torch.ones(192, dtype=torch.bool)
    keep[64 + 32 * c:96 + 32 * c] = False
    assert torch.equal(src[:, :, keep].view(torch.int16), before[:, :, keep].view(torch.int16))


@pytest.mark.parametrize('kernel', KERNELS_64, ids=KNAME.get)
@pytest.mark.parametrize('mode', (0, 2))
def test_exact_saturation(kernel, mode, cuda_device):
    """Activations +-2^10 and weights of one sign per output channel: interior sums reach 576 * 1024 / 8 = 73728 > 65504
    (all integers, exact in fp32); the fp16 store must saturate to +-65504 -- never inf or NaN -- while the smaller
    border sums stay exact."""
    bufs, checks = run_exact(kernel, 64, 64, 17, 33, mode=mode, operands='sat', seed=3)
    got = checks[0][1]
    assert bool((got == FP16_MAX).any()) and bool((got == -FP16_MAX).any()), 'no saturated output: the case lost its point'
    assert torch.isfinite(got).all()


@pytest.mark.parametrize('kernel', (WS_TMA, WS_CP, AUTO), ids=KNAME.get)
def test_exact_conv_first(kernel, cuda_device):
    """conv_first: 3 input channels in the NHWC32 layout nchw_to_nhwc32_kernel produces (channels 3..31 zero), padded
    to a 32-channel K slice with zero weights; fp32 trunk + feat copies (mode 3)."""
    H, W = 23, 50
    src, w, b = exact_operands(H, W, 32, 64, 3, 9, 'cuda')
    src[:, :, 3:] = 0
    v, *_ = conv_ref(src[:, :, :3].permute(2, 0, 1)[None].double(), w, b, False, True)
    df, df2 = (torch.full((H * W, 64), SENT32, device='cuda') for _ in range(2))
    st, used = run_layer(w, b, src, kernel, mode=3, dst_f=df, dst_f2=df2)
    expect_ran(st, used, kernel)
    torch.cuda.synchronize()
    assert used in (WS_TMA, WS_CP)
    for t in (df, df2):
        assert torch.equal(t.view(H, W, 64).permute(2, 0, 1), v.float())


def _decoder_layers():
    """(name, cout, cin, up, mode) of every convolution shape of k4_srnet_forward."""
    return [('conv_first', 64, 3, False, 6), ('rdb_conv1', 32, 64, False, 0), ('rdb_conv2', 32, 96, False, 0),
            ('rdb_conv3', 32, 128, False, 0), ('rdb_conv4', 32, 160, False, 5), ('rdb_conv5', 64, 192, False, 7),
            ('rdb_conv5_unfused', 64, 192, False, 1), ('conv_body', 64, 64, False, 2), ('conv_up', 64, 64, True, 0),
            ('conv_hr', 64, 64, False, 0), ('conv_last', 3, 64, False, 4)]


def test_auto_picks_k64_for_exactly_the_64_channel_layers(cuda_device):
    """K4_CONV_KERNEL_AUTO is the decoder's choice: conv3x3_k64_kernel for the 64-input-channel layers after the dense
    blocks (N = 64 or 16), conv3x3_ws_kernel (TMA producer) for every other one -- unless the environment switches
    K4_CONV_K64=0 / K4_CONV_NO_TMA=1 say otherwise."""
    use_k64 = os.environ.get('K4_CONV_K64', '1')[:1] != '0'
    ws = WS_CP if os.environ.get('K4_CONV_NO_TMA', '0')[:1] == '1' else WS_TMA
    seen = {}
    for name, cout, cin, up, mode in _decoder_layers():
        if mode >= 5:                       # the fused SFT modes: covered by test_sft_epilogues with AUTO below
            continue
        st, used, *_ = plain_layer(AUTO, cout, cin, 9, 27, mode=mode, up=up, lrelu=0.2 if mode == 0 else 0.0)
        assert st == OK
        seen[name] = used
        expect = K64 if (use_k64 and cin == 64 and npad_of(cout) in (16, 64)) else ws
        assert used == expect, (name, KNAME.get(used), KNAME[expect])
    print({k: KNAME[v] for k, v in seen.items()})


# ------------------------------------------------------------------------------------------------
# (b) random operands: the precision contract
# ------------------------------------------------------------------------------------------------
RANDOM_CFGS = ([(k, 64, 64, False) for k in KERNELS_64] + [(k, 64, 64, True) for k in KERNELS_64]
               + [(WS_TMA, 32, 160, False), (WS_CP, 32, 96, False), (WS_TMA, 64, 192, False), (WS_CP, 64, 192, False),
                  (K64, 16, 64, False), (WS_TMA, 16, 64, False)])


RANDOM_CASES = [(cfg, m) for cfg in RANDOM_CFGS for m in ((0, 0.2), (1, 0.0), (4, 0.0)) if not (cfg[0] == K64 and m[0] == 1)]


@pytest.mark.parametrize('cfg,mode_lrelu', RANDOM_CASES, ids=[f'{_cfg_id(c)}-mode{m[0]}' for c, m in RANDOM_CASES])
def test_random_layers_meet_the_precision_contract(cfg, mode_lrelu, cuda_device):
    """What DESIGN.md says is rounded and nothing else: activations and weights to fp16 (the sub-pixel layers: each
    phase-combined weight formed in fp64 from the fp32 weights and rounded to fp16 once, with a one-ulp allowance for a
    weight whose fp32 sum may round the other way), products accumulated in fp32.  Bar per element:
    |y - ref| <= 2^-16 * sum |a||w| (+ a few fp32 roundings of the epilogue, + half an fp16 ulp of ref for fp16
    outputs).  An operand held in bf16 or TF32 misses it by more than an order of magnitude.  (k64 runs only modes 0,
    2 and 4.)"""
    k, n, ci, up = cfg
    mode, lrelu = mode_lrelu
    cout = 3 if (mode == 4 and n == 16) else n
    st, used, bufs, checks, _ = plain_layer(k, cout, ci, 21, 53, mode=mode, lrelu=lrelu, up=up, rows=(2, 20),
                                            operands='random', seed=5 + ci)
    expect_ran(st, used, k)
    torch.cuda.synchronize()
    check_bound(checks, f'{_cfg_id(cfg)} mode {mode}')


PRETRAINED_LAYERS = [('conv_body', False, 0, K64), ('conv_up1', True, 0, K64), ('conv_up2', True, 0, WS_TMA),
                     ('conv_hr', False, 0, WS_CP), ('conv_last', False, 4, K64), ('body.0.rdb1.conv5', False, 1, WS_TMA),
                     ('body.1.rdb2.conv2', False, 0, WS_CP)]


@pytest.fixture(scope='module')
def pretrained_sd():
    from helpers import pretrained_sr_state_dict
    sd = pretrained_sr_state_dict()
    if sd is None:
        pytest.skip('oracle/_ref/RealESRNet_x4plus.pth missing')
    return sd


@pytest.mark.parametrize('layer', PRETRAINED_LAYERS, ids=lambda l: f'{l[0]}-{KNAME[l[3]]}')
def test_pretrained_magnitude_layers_meet_the_precision_contract(layer, pretrained_sd, cuda_device):
    """The same contract with the shipped checkpoint's weights (RealESRNet_x4plus)."""
    name, up, mode, k = layer
    w, b = pretrained_sd[name + '.weight'], pretrained_sd[name + '.bias']
    st, used, bufs, checks, _ = plain_layer(k, w.shape[0], w.shape[1], 19, 37, mode=mode, lrelu=0.2 if mode == 0 else 0.0,
                                            up=up, operands='random', seed=11, weight=(w, b))
    expect_ran(st, used, k)
    torch.cuda.synchronize()
    check_bound(checks, f'pretrained {name} ({KNAME[k]})')


# ------------------------------------------------------------------------------------------------
# (c) the fused SFT epilogues (modes 5-7)
# ------------------------------------------------------------------------------------------------
def sft_params(cout, seed, dev):
    """The four 1x1 convolutions of an SFT layer in k4_srnet_desc order (scale_conv0 w, b, scale_conv1 w, b, shift_conv0
    w, b, shift_conv1 w, b), at the reference's default-init magnitude."""
    g = torch.Generator().manual_seed(seed)
    shapes = [(32, 32), (32,), (cout, 32), (cout,), (32, 32), (32,), (cout, 32), (cout,)]
    ts = [(torch.rand(s, generator=g) * 2 - 1) * (1 / math.sqrt(32)) for s in shapes]
    return [t.contiguous().to(dev) for t in ts]


def sft_ref(p, c16):
    """fp64 SFT MLPs of one layer on the fp16 condition c16 [P, 32]: (scale + 1, shift) and their error bounds.  The hidden
    activation is rounded to fp16 as sft_hidden does (with a one-ulp allowance where the kernel's value may round the
    other way); weights fp16, biases fp32."""
    h16 = lambda t: t.half().double()
    W0 = h16(torch.cat([p[0], p[4]]))
    b0 = torch.cat([p[1], p[5]]).double()
    c = c16.double()
    hid = c @ W0.T + b0
    e_hid = 2.0 ** -16 * (c.abs() @ W0.abs().T) + FP32_EPS * hid.abs()
    hid = torch.where(hid > 0, hid, 0.2 * hid)
    slack = tie_slack(hid, e_hid)
    hq = h16(hid)
    out = []
    for (wi, bi, lo, plus) in ((2, 3, 0, 1.0), (6, 7, 32, 0.0)):
        W1 = h16(p[wi])
        hh, sl = hq[:, lo:lo + 32], slack[:, lo:lo + 32]
        y = hh @ W1.T + p[bi].double() + plus
        e = 2.0 ** -16 * (hh.abs() @ W1.abs().T) + sl @ W1.abs().T + FP32_EPS * (y.abs() + 1.0)
        out += [y, e]
    return out                                      # sc, e_sc, sh, e_sh


SFT_CASES = [  # (name, mode, cout, cin, H, W, rows, add_f, dst_f2, in_place)
    ('conv4_sft1', 5, 32, 160, 17, 33, None, False, False, True),
    ('conv4_sft1_window', 5, 32, 160, 40, 29, (3, 37), False, False, True),
    ('conv5_sft0', 6, 64, 192, 17, 33, None, True, False, False),
    ('conv_first_sft0', 6, 64, 3, 40, 29, (3, 37), False, True, False),
    ('conv5_rrdb_tail', 7, 64, 192, 17, 33, None, True, False, False),
    ('conv5_rrdb_tail_window', 7, 64, 192, 40, 29, (5, 6), True, False, False),
]


@pytest.mark.parametrize('case', SFT_CASES, ids=lambda c: c[0])
@pytest.mark.parametrize('kernel', (WS_TMA, AUTO), ids=KNAME.get)
def test_sft_epilogues(case, kernel, cuda_device):
    """The SFT layer(s) folded into the convolution's epilogue (mma.sync on the accumulator fragments), every output of
    each mode, against fp64: sft(x) = x * (scale + 1) + shift, scale / shift = W1 . lrelu(W0 . cond + b0) + b1 with fp16
    cond / W0 / W1, fp32 biases, the hidden activation rounded to fp16.  Mode 7 is the RRDB tail: u = sft(t) * 0.25 +
    x_in, then the next layer on u.  Bar: the element bound of the random-operand tests, carried through each stage."""
    name, mode, cout, cin, H, W, rows, with_add, with_f2, in_place = case
    dev = 'cuda'
    P = H * W
    ylo, yhi = rows if rows is not None else (0, H)
    cs = 192 if in_place else cpad_of(cin)
    src, w, b = random_operands(H, W, cs, cout, cin, 60 + mode, dev)
    if cin == 3:
        src[:, :, 3:] = 0
    g = torch.Generator().manual_seed(61)
    cond16 = (torch.randn(P, 32, generator=g) * 0.5).half().to(dev)
    sft1 = sft_params(cout, 62, dev)
    sft2 = sft_params(64, 63, dev) if mode == 7 else None
    a = src[:, :, :cin].permute(2, 0, 1)[None].double()
    v, S, _ = conv_ref(a, w, b, False, False)
    v, S = hwc(v), hwc(S)                                   # [P, cout]
    e_v = 2.0 ** -16 * S + FP32_EPS * v.abs()
    sc, e_sc, sh, e_sh = sft_ref(sft1, cond16)
    kw = dict(mode=mode, rows=rows, cond16=cond16, sft=sft1, sft2=sft2)
    checks = []
    sel = torch.zeros(H, W, dtype=torch.bool, device=dev)
    sel[ylo:yhi] = True
    sel = sel.view(-1)

    def half_out(got, ref, err):
        checks.append((got[sel], ref[sel], (err + 0.5 * ulp16(ref.abs() + err))[sel]))

    if mode == 5:
        before = src.clone()
        kw.update(lrelu=0.2, dst_h=src, dst_c0=160)
        v32 = v.float()
        act = torch.where(v32 > 0, v32, v32 * torch.tensor(0.2, dtype=torch.float32)).double()
        ref = act * sc + sh
        err = e_v * sc.abs() + act.abs() * e_sc + e_sh + FP32_EPS * (ref.abs() + (act * sc).abs())
        st, used = run_layer(w, b, src, kernel, **kw)
        expect_ran(st, used, kernel)
        torch.cuda.synchronize()
        half_out(src[:, :, 160:192].reshape(P, 32).double(), ref, err)
        keep = torch.ones(H, W, 192, dtype=torch.bool, device=dev)
        keep[ylo:yhi, :, 160:] = False
        assert torch.equal(src[keep].view(torch.int16), before[keep].view(torch.int16)), 'wrote outside rows / channels'
    else:
        scale = 1.0 if cin == 3 else 0.25
        add = trunk_operand(P, 64, dev, False) if with_add else None
        addr = add.double() if with_add else torch.zeros_like(v)
        t = v * scale + addr
        e_t = scale * e_v + FP32_EPS * (t.abs() + addr.abs())
        dst_f = torch.full((P, 64), SENT32, device=dev)
        dst_f2 = torch.full((P, 64), SENT32, device=dev) if with_f2 else None
        dst_h2 = torch.full((H, W, 96), SENT16, dtype=torch.float16, device=dev)
        kw.update(scale=scale, add_f=add, dst_f=dst_f, dst_f2=dst_f2, dst_h2=dst_h2, dst2_c0=16)
        m = t * sc + sh
        e_m = e_t * sc.abs() + t.abs() * e_sc + e_sh + FP32_EPS * (m.abs() + (t * sc).abs())
        if mode == 6:
            f_ref, f_err, h_ref, h_err = t, e_t, m, e_m
        else:
            x_in = trunk_operand(P, 65, dev, False)
            kw.update(add_f2=x_in, scale2=0.25)
            u = m * 0.25 + x_in.double()
            e_u = 0.25 * e_m + FP32_EPS * (u.abs() + x_in.double().abs())
            sc2, e_sc2, sh2, e_sh2 = sft_ref(sft2, cond16)
            m2 = u * sc2 + sh2
            f_ref, f_err = u, e_u
            h_ref, h_err = m2, e_u * sc2.abs() + u.abs() * e_sc2 + e_sh2 + FP32_EPS * (m2.abs() + (u * sc2).abs())
        st, used = run_layer(w, b, src, kernel, **kw)
        expect_ran(st, used, kernel)
        torch.cuda.synchronize()
        for d in [dst_f] + ([dst_f2] if with_f2 else []):
            checks.append((d.double()[sel], f_ref[sel], f_err[sel]))
            assert bool((d[~sel] == SENT32).all()), 'trunk rows outside the window written'
        half_out(dst_h2[:, :, 16:80].reshape(P, 64).double(), h_ref, h_err)
        outside = torch.ones(H, W, 96, dtype=torch.bool, device=dev)
        outside[ylo:yhi, :, 16:80] = False
        assert bool((dst_h2[outside] == SENT16).all()), 'dst_h2 written outside rows / channels'
    check_bound([(f'out{i}', g_, r_, e_) for i, (g_, r_, e_) in enumerate(checks)], f'sft {name} ({KNAME[kernel]})')
    if kernel == AUTO:
        ws = WS_CP if os.environ.get('K4_CONV_NO_TMA', '0')[:1] == '1' else WS_TMA
        assert used == ws


# ------------------------------------------------------------------------------------------------
# (d) CondNet
# ------------------------------------------------------------------------------------------------
MMA, FP32 = _lib.K4_SR_KERNEL_MMA, _lib.K4_SR_KERNEL_FP32
PKNAME = {_lib.K4_SR_KERNEL_AUTO: 'auto', MMA: 'mma', FP32: 'fp32'}
U = 2.0 ** -24                   # unit roundoff of fp32
GAMMA_TC = 17 * 2.0 ** -23       # one mma.sync instruction, relative to S (test_gpu_march_mlp.py)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def condnet_params(seed, dev, scale=1.0):
    """CondNet.0 (64x1x3x3), .2, .4 (64x64x1x1), .6 (32x64x1x1), weight and bias each, as nn.Conv2d initialises them
    (uniform in +-1 / sqrt(fan_in)), times `scale`."""
    g = torch.Generator().manual_seed(seed)
    ts = []
    for shape, fan in (((64, 1, 3, 3), 9), ((64, 64, 1, 1), 64), ((64, 64, 1, 1), 64), ((32, 64, 1, 1), 64)):
        bound = scale / math.sqrt(fan)
        ts += [(torch.rand(shape, generator=g) * 2 - 1) * bound, (torch.rand(shape[0], generator=g) * 2 - 1) * bound]
    return [t.contiguous().to(dev) for t in ts]


def depth_map(H, W, seed, dev):
    """A depth-like condition in [0, 1]: a ramp, flat plateaus with sharp edges, a noisy patch, exact 0 and 1 flats."""
    g = torch.Generator().manual_seed(seed)
    y, x = torch.linspace(0, 1, H)[:, None], torch.linspace(0, 1, W)[None]
    d = (0.3 + 0.5 * x * (1 - 0.5 * y)).expand(H, W).clone()
    for _ in range(4):
        y0, x0 = int(torch.randint(0, H, (1,), generator=g)), int(torch.randint(0, W, (1,), generator=g))
        d[y0:y0 + max(1, H // 3), x0:x0 + max(1, W // 3)] = torch.rand(1, generator=g).item()
    d[H // 2:, W // 2:W // 2 + max(1, W // 4)] = torch.rand(H - H // 2, min(W, W // 2 + max(1, W // 4)) - W // 2, generator=g)
    d[:max(1, H // 5)] = 1.0
    d[:, :W // 6] = 0.0
    return d.clamp(0, 1).contiguous().to(dev)


def run_condnet(params, cond_in, kernel, rows=None):
    """One k4_testing_condnet call into sentinel-filled cond_out [P, 32] / cond16 [P, 32].  Returns them and the kernel."""
    H, W = cond_in.shape
    out = torch.full((H * W, 32), SENT32, device=cond_in.device)
    c16 = torch.full((H * W, 32), SENT16, dtype=torch.float16, device=cond_in.device)
    a = _lib.CondnetTestArgs()
    a.h_condnet = _sft_ptrs(params)
    a.d_cond_in, a.H, a.W = cond_in.data_ptr(), H, W
    a.y_lo, a.y_hi = rows if rows is not None else (0, H)
    a.d_cond_out, a.d_cond16, a.kernel = out.data_ptr(), c16.data_ptr(), kernel
    used = C.c_int32(-9)
    st = _lib.lib.k4_testing_condnet(C.byref(a), C.byref(used), _stream())
    assert st == OK, f'k4_testing_condnet -> {st} ({_lib.lib.k4_status_string(st).decode()}) for {PKNAME[kernel]}'
    if kernel != _lib.K4_SR_KERNEL_AUTO:
        assert used.value == kernel, (PKNAME[kernel], used.value)
    return out, c16, used.value


def lrelu(t):
    return torch.where(t > 0, t, 0.2 * t)


def condnet_ref(p, cond_in, kernel):
    """fp64 CondNet on the whole map: conv3x3 with zero padding, then the three 1x1 layers, LeakyReLU 0.2 between.
    Returns the output [P, 32], the per-element bound E of `kernel` [P, 32] and the largest |hidden activation|.

    The bound is carried layer to layer: e_{l+1} = gamma_l * S_{l+1} + |W_{l+1}| e_l, S = |b| + sum |a| |w| over the
    layer's products, with |a| taken as |a_ref| + e_l.  LeakyReLU is 1-Lipschitz; its fp32 multiply by 0.2f (not 0.2)
    adds at most 2u |z|.  u = 2^-24.
      * Layer 0 (both kernels): an FFMA chain of 9 products from the bias, 10u * S.
      * fp32 kernel, 1x1 layers: an FFMA chain of 64 products, 65u * S.
      * mma kernel, 1x1 layers: x = hi + lo with hi = fp16(x), lo = fp16(x - hi) for activations and weights alike:
        |x - hi - lo| <= 2^-22 |x| + 2^-25 (a lo part below 2^-14 is an fp16 subnormal, spaced 2^-24 -- the case of
        |x| < 2^-3, so of most 1x1 weights, bound 1/8) and |lo| <= 2^-11 |x| + 2^-24.  The product drops lo_a lo_w and
        the two representation errors; its S counts the three fp16 products.  Four k16 steps of three MMAs are 12
        instructions, each within 17 * 2^-23 * S (a truncating fp32 accumulation of 16 exact products, the model of
        test_gpu_march_mlp.py): 12 * 17 * 2^-23 * S, about 2^-15.3 S.
    Carried through |W| (sum |w| is about 4 per row at nn.Conv2d initialisation) the output bound of default weights
    ends near 2^-10 of the output scale: it catches a wrong tap, padding row, window or layer, but not a lost lo term of
    random sign (about 2^-15 S); test_condnet_exact_operands checks the lo terms bit for bit."""
    W0, b0 = p[0].double(), p[1].double()
    c = cond_in.double()[None, None]
    z = hwc(F.conv2d(c, W0, b0, padding=1)[0])
    E = 10 * U * (hwc(F.conv2d(c.abs(), W0.abs(), padding=1)[0]) + b0.abs())
    hmax = 0.0
    for i in (2, 4, 6):
        a = lrelu(z)
        D = E + 2 * U * (z.abs() + E)
        hmax = max(hmax, a.abs().max().item())
        Wl, bl = p[i].double().view(p[i].shape[0], 64), p[i + 1].double()
        av, aw = a.abs() + D, Wl.abs()
        z = a @ Wl.T + bl
        if kernel == FP32:
            E = D @ aw.T + 65 * U * (av @ aw.T + bl.abs())
        else:
            ev, lv = 2.0 ** -22 * av + 2.0 ** -25, 2.0 ** -11 * av + 2.0 ** -24
            ew, lw = 2.0 ** -22 * aw + 2.0 ** -25, 2.0 ** -11 * aw + 2.0 ** -24
            split = lv @ lw.T + av @ ew.T + ev @ aw.T + ev @ ew.T
            S = av @ aw.T + av @ lw.T + lv @ aw.T + bl.abs()
            E = D @ aw.T + split + 12 * GAMMA_TC * S
    return z, E, hmax


def check_condnet_outputs(out, c16, ref, bound, rows, H, W, label):
    """cond_out within the bound (or equal to ref when bound is None) on the window's rows; cond16 is bitwise the saturated
    fp16 rounding of the kernel's own cond_out; every row outside the window keeps its sentinel."""
    ylo, yhi = rows if rows is not None else (0, H)
    win = slice(ylo * W, yhi * W)
    got = out[win]
    if bound is None:
        check_exact([('cond_out', got, ref[win].float(), None)])
        worst = 0.0
    else:
        worst = check_bound([('cond_out', got, ref[win], bound[win])], label)
    want16 = got.clamp(-FP16_MAX, FP16_MAX).half()
    assert torch.equal(c16[win].view(torch.int16), want16.view(torch.int16)), 'cond16 is not the saturated fp16 rounding of cond_out'
    outside = torch.ones(H * W, dtype=torch.bool, device=out.device)
    outside[win] = False
    assert bool((out[outside] == SENT32).all()) and bool((c16[outside] == SENT16).all()), 'rows outside the window written'
    return worst


CONDNET_CASES = [  # (name, H, W, rows, weight scale)
    ('1x1', 1, 1, None, 1.0), ('1x7', 1, 7, None, 1.0), ('7x1', 7, 1, None, 4.0), ('19x13', 19, 13, None, 1.0),
    ('19x13_w4', 19, 13, None, 4.0), ('rows5-6', 40, 29, (5, 6), 1.0), ('rows3-37', 40, 29, (3, 37), 4.0),
    ('rows16-33', 40, 29, (16, 33), 1.0),
]


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
@pytest.mark.parametrize('case', CONDNET_CASES, ids=lambda c: c[0])
def test_condnet_meets_its_element_bound(case, kernel, cuda_device):
    """CondNet on depth-like maps (flats, sharp edges, noise) with nn.Conv2d-initialised weights x1 and x4, at shapes
    down to 1x1, P = 247 (not a multiple of 16) and row windows strictly inside the map, whose edge rows must see the
    real neighbour rows above and below: every output within the bound of condnet_ref."""
    name, H, W, rows, scale = case
    p = condnet_params(70 + H + W, 'cuda', scale)
    cond_in = depth_map(H, W, 71 + H, 'cuda')
    ref, E, _ = condnet_ref(p, cond_in, kernel)
    out, c16, _ = run_condnet(p, cond_in, kernel, rows)
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, E, rows, H, W, f'condnet {name} ({PKNAME[kernel]})')


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
def test_condnet_grid_stride_wraps(kernel, cuda_device):
    """More than 3 x (4 * SM-count CTAs x 64 pixels): the mma kernel's capped grid strides over the map more than three
    times (the fp32 kernel takes one thread per pixel)."""
    W = 331
    H = 3 * 4 * sm_count() * 64 // W + 3
    assert H * W > 3 * 4 * sm_count() * 64
    p = condnet_params(80, 'cuda')
    cond_in = depth_map(H, W, 81, 'cuda')
    ref, E, _ = condnet_ref(p, cond_in, kernel)
    out, c16, _ = run_condnet(p, cond_in, kernel, (1, H))
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, E, (1, H), H, W, f'condnet {H}x{W} ({PKNAME[kernel]})')


def exact_condnet_params(seed, dev):
    """Non-negative dyadic CondNet weights for test_condnet_exact_operands: W0 j/8 (j <= 2), 1x1 rows of two non-zero
    weights -- CondNet.2 of 12 significant bits, (2^11 + odd) * 2^-15, so each has an fp16 lo part; CondNet.4 and .6
    exactly 1/2 -- and biases m/64 (m <= 16)."""
    g = torch.Generator().manual_seed(seed)

    def sparse(n_out, value):
        w = torch.zeros(n_out, 64)
        for o in range(n_out):
            w[o, torch.randperm(64, generator=g)[:2]] = value(2)
        return w.view(n_out, 64, 1, 1)

    bias = lambda n: torch.randint(0, 17, (n,), generator=g) / 64.0
    ts = [torch.randint(0, 3, (64, 1, 3, 3), generator=g) / 8.0, bias(64),
          sparse(64, lambda n: (2 ** 11 + 2 * torch.randint(0, 2 ** 10, (n,), generator=g) + 1) * 2.0 ** -15), bias(64),
          sparse(64, lambda n: torch.full((n,), 0.5)), bias(64),
          sparse(32, lambda n: torch.full((n,), 0.5)), bias(32)]
    return [t.contiguous().to(dev) for t in ts]


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
def test_condnet_exact_operands(kernel, cuda_device):
    """Operands whose every sum is exact in fp32 and whose activations fit the mma kernel's 22-bit hi + lo split exactly:
    the condition on the 1/2 grid, so layer 0's outputs lie on the 2^-4 grid below 2.75 (7 bits, no lo part); CondNet.2
    weights with lo parts make layer 1's outputs 19-bit values (2^-19 grid, < 1), and the halving 1x1 layers keep 20 and
    21 bits.  Every lo x lo product is zero (layer 1: no activation lo parts; layers 2, 3: no weight lo parts), so both
    kernels must EQUAL the fp64 reference: a lost al * Wh term (layers 2, 3), a lost weight lo part (layer 1), a moved
    tap or a wrong padding row is a non-zero difference."""
    H, W = 23, 37
    p = exact_condnet_params(85, 'cuda')
    cond_in = ((depth_map(H, W, 86, 'cuda') * 2).round() / 2).contiguous()
    ref, _, _ = condnet_ref(p, cond_in, kernel)
    # the case's premises, checked on the reference's activations
    z = hwc(F.conv2d(cond_in.double()[None, None], p[0].double(), p[1].double(), padding=1)[0])
    for i in (2, 4, 6):
        hi = z.half().double()
        assert torch.equal((z - hi).half().double(), z - hi), 'an activation does not fit the hi + lo split'
        if i > 2:
            assert bool(((z - hi) != 0).any()), 'no activation lo part: the case lost its point'
        z = z @ p[i].double().view(-1, 64).T + p[i + 1].double()
        assert torch.equal(z.float().double(), z)
    w2 = p[2].view(64, 64)
    assert bool(((w2 - w2.half().float()) != 0).sum() > 32), 'no weight lo part: the case lost its point'
    rows = (3, 20)
    out, c16, _ = run_condnet(p, cond_in, kernel, rows)
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, None, rows, H, W, f'condnet exact ({PKNAME[kernel]})')


def test_condnet_auto_follows_the_env_switch_per_call(monkeypatch, cuda_device):
    """K4_SR_KERNEL_AUTO is the decoder's choice: the mma kernel, or the fp32 kernel while K4_CONDNET_FP32=1 (read per call)."""
    p = condnet_params(87, 'cuda')
    cond_in = depth_map(5, 9, 88, 'cuda')
    monkeypatch.delenv('K4_CONDNET_FP32', raising=False)
    assert run_condnet(p, cond_in, _lib.K4_SR_KERNEL_AUTO)[2] == MMA
    monkeypatch.setenv('K4_CONDNET_FP32', '1')
    assert run_condnet(p, cond_in, _lib.K4_SR_KERNEL_AUTO)[2] == FP32


# ------------------------------------------------------------------------------------------------
# (e) the standalone SFT pass (K4_SR_FUSE_SFT=0, and every decoder call without TMA)
# ------------------------------------------------------------------------------------------------
RES_SCALE = float(torch.tensor(0.2, dtype=torch.float32))      # what the kernel multiplies by


def run_sft_pass(p, cout, cond, kernel, *, x_f=None, x_h=None, xh_c0=0, dst_h=None, dst_c0=0, dst_f=None, res_f=None,
                 res_scale=0.0, p0=0, P=1):
    """One k4_testing_sft call.  x_h / dst_h: fp16 [pixels, cstride]; x_f / dst_f / res_f: fp32 [pixels, 64]."""
    a = _lib.SftTestArgs()
    a.h_sft, a.cout, a.kernel, a.d_cond = _sft_ptrs(p), cout, kernel, cond.data_ptr()
    a.d_x_f, a.d_x_h, a.xh_cstride, a.xh_c0 = _ptr(x_f), _ptr(x_h), (x_h.shape[-1] if x_h is not None else 0), xh_c0
    a.d_dst_h, a.dst_cstride, a.dst_c0 = _ptr(dst_h), (dst_h.shape[-1] if dst_h is not None else 0), dst_c0
    a.d_dst_f, a.d_res_f, a.res_scale, a.p0, a.P = _ptr(dst_f), _ptr(res_f), res_scale, p0, P
    used = C.c_int32(-9)
    st = _lib.lib.k4_testing_sft(C.byref(a), C.byref(used), _stream())
    assert st == OK, f'k4_testing_sft -> {st} ({_lib.lib.k4_status_string(st).decode()}) for {PKNAME[kernel]}'
    if kernel != _lib.K4_SR_KERNEL_AUTO:
        assert used.value == kernel, (PKNAME[kernel], used.value)
    return used.value


def sft_ref32(p, cond):
    """fp64 SFT MLPs of one layer on the fp32 condition and fp32 weights, with the fp32 kernel's bounds: FFMA chains of
    32 products from the bias (33u * S), LeakyReLU's multiply by 0.2f (2u), scale + 1 (u).  Returns sc (scale + 1),
    e_sc, sh, e_sh like sft_ref."""
    c = cond.double()
    W0, b0 = torch.cat([p[0], p[4]]).double(), torch.cat([p[1], p[5]]).double()
    hid = c @ W0.T + b0
    e = 33 * U * (c.abs() @ W0.abs().T + b0.abs())
    a = lrelu(hid)
    e = e + 2 * U * (hid.abs() + e)
    out = []
    for (wi, bi, lo, plus) in ((2, 3, 0, 1.0), (6, 7, 32, 0.0)):
        W1, b1 = p[wi].double(), p[bi].double()
        aa, ee = a[:, lo:lo + 32], e[:, lo:lo + 32]
        y = aa @ W1.T + b1 + plus
        ey = ee @ W1.abs().T + 33 * U * ((aa.abs() + ee) @ W1.abs().T + b1.abs()) + plus * U * (y.abs() + 1.0)
        out += [y, ey]
    return out


# (name, what the decoder runs it on): the four I/O forms of run_sft in srnet_forward_roi_impl, each with a row window of
# a 40 x 29 map as win() gives it
SFT_FORMS = [('trunk_to_cat', (0, 40)), ('cat_in_place', (13, 27)), ('rrdb_tail_aliased', (14, 26)), ('sbody', (9, 31))]


def sft_pass_case(form, cout, kernel, H, W, rows, seed):
    """Run one form and return [(name, got, ref, bound)] plus the sentinel / untouched checks already asserted."""
    dev = 'cuda'
    Pall = H * W
    p0, P = rows[0] * W, (rows[1] - rows[0]) * W
    win = slice(p0, p0 + P)
    g = torch.Generator().manual_seed(seed)
    p = sft_params(cout, seed + 1, dev)
    cond = (torch.randn(Pall, 32, generator=g) * 0.5).to(dev)
    if kernel == FP32:
        sc, e_sc, sh, e_sh = sft_ref32(p, cond[win])
    else:
        sc, e_sc, sh, e_sh = sft_ref(p, cond[win].clamp(-FP16_MAX, FP16_MAX).half())
    kw = dict(p0=p0, P=P)
    if form == 'cat_in_place':
        c0 = 192 - cout
        buf = (torch.rand(Pall, 192, generator=g) * 3 - 1).half().to(dev)
        x = buf[win, c0:c0 + cout].double()
        kw.update(x_h=buf, xh_c0=c0, dst_h=buf, dst_c0=c0)
    else:
        xf = trunk_operand(Pall, seed + 2, dev, False)
        x = xf[win, :cout].double()
        kw['x_f'] = xf
    y = x * sc + sh
    e_y = x.abs() * e_sc + e_sh + FP32_EPS * (y.abs() + (x * sc).abs())
    if form == 'rrdb_tail_aliased':
        buf = trunk_operand(Pall, seed + 3, dev, False)
        c0, cs = 0, 64
        r = buf[win, :cout].double()
        kw.update(dst_f=buf, res_f=buf, res_scale=RES_SCALE)
    elif form != 'cat_in_place':
        c0, cs = (0, 192) if form == 'trunk_to_cat' else (0, 64)
        buf = torch.full((Pall, cs), SENT16, dtype=torch.float16, device=dev)
        kw.update(dst_h=buf, dst_c0=c0)
    before = buf.clone()
    used = run_sft_pass(p, cout, cond, kernel, **kw)
    torch.cuda.synchronize()
    got = buf[win, c0:c0 + cout].double()
    if form == 'rrdb_tail_aliased':
        ref = y * RES_SCALE + r
        bound = RES_SCALE * e_y + FP32_EPS * ((y * RES_SCALE).abs() + ref.abs())
    else:
        ref, bound = y, e_y + 0.5 * ulp16(y.abs() + e_y)
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[win, c0:c0 + cout] = False
    assert torch.equal(buf[keep].view(torch.int32 if buf.dtype == torch.float32 else torch.int16),
                       before[keep].view(torch.int32 if buf.dtype == torch.float32 else torch.int16)), \
        'wrote outside the pixel window / channels'
    return [(form, got, ref, bound)], used


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
@pytest.mark.parametrize('cout', (32, 64))
@pytest.mark.parametrize('form', SFT_FORMS, ids=lambda f: f[0])
def test_sft_pass_meets_its_element_bound(form, cout, kernel, cuda_device):
    """One SFT layer as its own pass, in each of the decoder's four I/O forms: fp32 trunk in -> fp16 concat channels 0..;
    fp16 in place at the top channels of the 192-stride concat buffer; fp32 out aliased with the fp32 residual, y * 0.2 +
    res (the RRDB tail); fp32 trunk in -> the 64-stride sbody.  Pixel windows [p0, p0 + P) with P = 14 * 29, 22 * 29, ...
    (not multiples of 16).  mma kernel: sft_ref on the saturated fp16 condition (fp16 weights, hidden activation rounded
    to fp16), carried through x * (scale + 1) + shift and the residual; fp32 kernel: sft_ref32.  fp16 outputs: + half an
    fp16 ulp of the unrounded value.  Everything outside the window and the layer's channels keeps its bytes."""
    name, rows = form
    checks, _ = sft_pass_case(name, cout, kernel, 40, 29, rows, 100 + cout)
    check_bound(checks, f'sft pass {name} cout {cout} ({PKNAME[kernel]})')


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
@pytest.mark.parametrize('cout', (32, 64))
def test_sft_pass_grid_stride_wraps(cout, kernel, cuda_device):
    """More than 3 x (8 * SM-count CTAs x 64 pixels): the mma kernel's capped grid strides over the window more than
    three times."""
    W = 331
    H = 3 * 8 * sm_count() * 64 // W + 4
    assert (H - 3) * W > 3 * 8 * sm_count() * 64
    checks, _ = sft_pass_case('rrdb_tail_aliased', cout, kernel, H, W, (2, H - 1), 110 + cout)
    check_bound(checks, f'sft pass {H}x{W} cout {cout} ({PKNAME[kernel]})')


def test_sft_pass_auto_is_the_decoders_choice(cuda_device):
    """K4_SR_KERNEL_AUTO runs the mma kernel, or the fp32 kernel when the process started with K4_SFT_FP32 set."""
    _, used = sft_pass_case('sbody', 64, _lib.K4_SR_KERNEL_AUTO, 3, 29, (1, 3), 120)
    assert used == (FP32 if 'K4_SFT_FP32' in os.environ else MMA)


# ------------------------------------------------------------------------------------------------
# (f) fp16 saturation of the condition
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
def test_condnet_outputs_beyond_fp16_saturate_cond16(kernel, cuda_device):
    """CondNet.6 scaled by a power of two (its weights stay below 65504) so that some conditions exceed the fp16 range
    while every hidden activation stays inside it: cond_out still meets the element bound, cond16 holds +-65504 (the
    operand the fused SFT epilogues read), and a fused-SFT convolution on that cond16 stays finite."""
    H, W = 19, 13
    p = condnet_params(130, 'cuda', 4.0)
    cond_in = depth_map(H, W, 131, 'cuda')
    f = 2.0 ** math.floor(math.log2(FP16_MAX / p[6].abs().max().item()))
    p[6], p[7] = p[6] * f, p[7] * f
    ref, E, hmax = condnet_ref(p, cond_in, kernel)
    assert hmax < FP16_MAX and bool((ref > FP16_MAX).any()) and bool((ref < -FP16_MAX).any()), 'the case lost its point'
    out, c16, _ = run_condnet(p, cond_in, kernel)
    torch.cuda.synchronize()
    check_condnet_outputs(out, c16, ref, E, None, H, W, f'condnet saturating ({PKNAME[kernel]})')
    assert bool((c16 == FP16_MAX).any()) and bool((c16 == -FP16_MAX).any())
    src, w, b = random_operands(H, W, 64, 64, 64, 132, 'cuda')
    dst_f = torch.full((H * W, 64), SENT32, device='cuda')
    dst_h2 = torch.full((H, W, 64), SENT16, dtype=torch.float16, device='cuda')
    st, used = run_layer(w, b, src, AUTO, mode=6, dst_f=dst_f, dst_h2=dst_h2, cond16=c16, sft=sft_params(64, 133, 'cuda'))
    expect_ran(st, used, AUTO)
    torch.cuda.synchronize()
    assert torch.isfinite(dst_h2).all(), 'the fused SFT epilogue turned a saturated condition into inf / NaN'


@pytest.mark.parametrize('kernel', (MMA, FP32), ids=PKNAME.get)
def test_condnet_hidden_activations_beyond_fp16_stay_finite(kernel, cuda_device):
    """CondNet.0 scaled by 2^17: layer-0 activations reach about 2e5, beyond fp16 and beyond 65504 + 65504 (so the mma
    kernel's hi part and its lo part would both overflow without saturation).  Both kernels' outputs stay finite."""
    H, W = 19, 13
    p = condnet_params(140, 'cuda')
    p[0], p[1] = p[0] * 2.0 ** 17, p[1] * 2.0 ** 17
    cond_in = depth_map(H, W, 141, 'cuda')
    _, _, hmax = condnet_ref(p, cond_in, kernel)
    assert hmax > 2 * FP16_MAX, 'the case lost its point'
    out, c16, _ = run_condnet(p, cond_in, kernel)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(c16).all()
    assert torch.equal(c16.view(torch.int16), out.clamp(-FP16_MAX, FP16_MAX).half().view(torch.int16))


# ------------------------------------------------------------------------------------------------
# the A/B environment switches, at network level
# ------------------------------------------------------------------------------------------------
_CHILD = r'''
import sys
import torch
sys.path[:0] = [sys.argv[1], sys.argv[1] + '/4k-nerf_b200']
import k4nerf
from oracle import sftnet
n = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
n.load_state_dict(sftnet.random_state_dict(seed=3))
n = n.cuda()
g = torch.Generator().manual_seed(5)
x = torch.rand(1, 3, 19, 13, generator=g)
c = torch.rand(1, 1, 19, 13, generator=g)
torch.save(n(x.cuda(), c.cuda()).cpu(), sys.argv[2])
'''
SWITCHES = ('K4_CONV_K64', 'K4_CONV_NO_TMA', 'K4_SR_PDL', 'K4_SFT_FP32', 'K4_SR_FUSE_SFT', 'K4_CONDNET_FP32')
ENVS = [('default', {}), ('no_k64', {'K4_CONV_K64': '0'}), ('no_tma', {'K4_CONV_NO_TMA': '1'}), ('no_pdl', {'K4_SR_PDL': '0'}),
        ('sft_fp32', {'K4_SFT_FP32': '1', 'K4_SR_FUSE_SFT': '0'}), ('condnet_fp32', {'K4_CONDNET_FP32': '1'})]


def test_decoder_environment_switches_in_child_processes(tmp_path, cuda_device):
    """The decoder's A/B switches K4_CONV_K64, K4_CONV_NO_TMA, K4_SR_PDL and K4_SFT_FP32 are latched in function-local
    statics at the first decoder call of a process, so a test cannot flip them in its own interpreter: each environment
    runs the seeded SFTNet forward of test_gpu_sftnet.py in a child interpreter.  Every run reaches 60 dB against
    oracle.sftnet; without programmatic dependent launch the result is bit-identical (PDL changes scheduling, not
    arithmetic); the other paths agree with the default within the fused-vs-unfused bar (66 dB)."""
    from oracle import pipeline, sftnet
    base = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    flags = ['-s'] if sys.flags.no_user_site else []
    outs = {}
    for name, env in ENVS:
        path = tmp_path / f'{name}.pt'
        r = subprocess.run([sys.executable, *flags, '-c', _CHILD, ROOT, str(path)], env=dict(base, **env), cwd=str(tmp_path),
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (name, r.stderr[-3000:])
        outs[name] = torch.load(path)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1, 3, 19, 13, generator=g)
    c = torch.rand(1, 1, 19, 13, generator=g)
    ref = sftnet.sftnet_forward(sftnet.random_state_dict(seed=3), x, c)
    for name, y in outs.items():
        p, pd = pipeline.psnr(y, ref), pipeline.psnr(y, outs['default'])
        print(f'{name}: {p:.2f} dB vs oracle, {pd:.2f} dB vs default')
        assert p >= 60.0, (name, p)
        if name == 'no_pdl':
            assert torch.equal(y, outs['default'])
        elif name != 'default':
            assert pd >= 66.0, (name, pd)
