"""Checkpoint helpers with the reference names (lib/utils.py:53-66), PSNR (lib/utils.py:18-19) and SSIM (lib/utils.py:88-134)."""
import numpy as np
import torch


def load_model(model_class, ckpt_path):
    """``model_class(**ckpt['model_kwargs']); load_state_dict`` -- the reference's .tar layout
    ``{global_step, model_kwargs, model_state_dict, optimizer_state_dict}`` loads unchanged."""
    ckpt = torch.load(ckpt_path, map_location='cpu', weights_only=False)
    model = model_class(**ckpt['model_kwargs'])
    model.load_state_dict(ckpt['model_state_dict'])
    return model


def mse2psnr(x):
    return -10. * torch.log10(x)


def to8b(x):
    return (255 * np.clip(x, 0, 1)).astype(np.uint8)


def _ssim_window(filter_size, filter_sigma):
    """The normalised 1-D Gaussian taps of ``rgb_ssim`` (lib/utils.py:99-104), for both of its paths."""
    half = filter_size // 2
    offs = np.arange(filter_size) - half + (2 * half - filter_size + 1) / 2      # centred taps (even sizes: half-pixel shift)
    win = np.exp(-0.5 * (offs / filter_sigma) ** 2)
    win /= win.sum()
    return win


def _is_cuda(x):
    return isinstance(x, torch.Tensor) and x.is_cuda


def _rgb_ssim_cuda(img0, img1, win, c1, c2, return_map):
    """``rgb_ssim`` of CUDA tensors by ``k4_op_rgb_ssim`` (csrc/k4_metrics.cu), read in place through their strides.
    A pair of fp32 images stays fp32; any other pair is promoted to fp64 (exactly, as numpy's ``asarray``)."""
    import ctypes as C
    from . import _lib
    if not (_is_cuda(img0) and _is_cuda(img1) and img0.device == img1.device):
        raise RuntimeError(f'rgb_ssim: img0 and img1 must be on one device (got {getattr(img0, "device", "numpy")} and '
                           f'{getattr(img1, "device", "numpy")})')
    assert img0.ndim == 3 and img0.shape[-1] == 3 and img0.shape == img1.shape
    H, W, f = img0.shape[0], img0.shape[1], len(win)
    if not 1 <= f <= 31:
        raise ValueError(f'rgb_ssim: filter_size must be in 1..31 on the GPU (got {f})')
    if H < f or W < f:
        raise ValueError('window shape cannot be larger than input array shape')
    img0, img1 = img0.detach(), img1.detach()
    if img0.dtype == img1.dtype == torch.float32:
        dtype = 0                                                   # K4_DTYPE_F32
    else:
        dtype = 1                                                   # K4_DTYPE_F64
        img0, img1 = img0.to(torch.float64), img1.to(torch.float64)
    dev = img0.device
    with torch.cuda.device(dev):
        ws = torch.empty(_lib.lib.k4_op_rgb_ssim_workspace_bytes(H, W, f), dtype=torch.uint8, device=dev)
        mean = torch.empty((), dtype=torch.float64, device=dev)
        ssim_map = torch.empty((H - f + 1, W - f + 1, 3), dtype=torch.float64, device=dev) if return_map else None
        strides = [(C.c_int64 * 3)(*t.stride()) for t in (img0, img1)]
        h_win = (C.c_double * f)(*win.tolist())
        _lib.check(_lib.lib.k4_op_rgb_ssim(
            C.c_void_p(img0.data_ptr()), C.c_void_p(img1.data_ptr()), dtype, H, W, strides[0], strides[1], h_win, f,
            float(c1), float(c2), None if ssim_map is None else C.c_void_p(ssim_map.data_ptr()), C.c_void_p(mean.data_ptr()),
            C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), 'k4_op_rgb_ssim')
    return ssim_map if return_map else float(mean.item())


def rgb_ssim(img0, img1, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, return_map=False):
    """Mean structural similarity of two ``[H, W, 3]`` images as ``lib/utils.py:88-134`` (the mip-NeRF evaluation
    variant) defines it: per channel, local means / variances / covariance under a ``filter_size`` Gaussian window
    (sigma ``filter_sigma``), 'valid' positions only, variances clipped at 0 and the covariance at the Cauchy-Schwarz
    bound, ``c1 = (k1 max_val)^2``, ``c2 = (k2 max_val)^2``.  Every operation is in fp64.

    CUDA tensors (both on one device) are scored on the GPU by ``k4_op_rgb_ssim`` (``filter_size`` up to 31); any view
    is read in place, e.g. ``rgb_ssim(sr.permute(1, 2, 0), gt, 1)`` for a ``[3, H, W]`` frame.  The mean comes back as a
    float (one 8-byte read), the map (``return_map``) as a CUDA fp64 tensor.  Numpy arrays and CPU tensors take the
    numpy path.  Both give the same values up to the order of the window sums (about 1e-15)."""
    if _is_cuda(img0) or _is_cuda(img1):
        c1, c2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
        return _rgb_ssim_cuda(img0, img1, _ssim_window(filter_size, filter_sigma), c1, c2, return_map)
    img0 = np.asarray(img0, dtype=np.float64)
    img1 = np.asarray(img1, dtype=np.float64)
    assert img0.ndim == 3 and img0.shape[-1] == 3 and img0.shape == img1.shape
    win = _ssim_window(filter_size, filter_sigma)

    def blur(z):          # separable 'valid' Gaussian window over the two image axes
        z = np.tensordot(np.lib.stride_tricks.sliding_window_view(z, filter_size, axis=0), win[::-1], axes=([-1], [0]))
        return np.tensordot(np.lib.stride_tricks.sliding_window_view(z, filter_size, axis=1), win[::-1], axes=([-1], [0]))

    m0, m1 = blur(img0), blur(img1)
    v0 = np.maximum(blur(img0 * img0) - m0 * m0, 0.0)
    v1 = np.maximum(blur(img1 * img1) - m1 * m1, 0.0)
    cov = blur(img0 * img1) - m0 * m1
    cov = np.sign(cov) * np.minimum(np.sqrt(v0 * v1), np.abs(cov))
    c1, c2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
    ssim_map = ((2 * m0 * m1 + c1) * (2 * cov + c2)) / ((m0 * m0 + m1 * m1 + c1) * (v0 + v1 + c2))
    return ssim_map if return_map else float(ssim_map.mean())


# ------------------------------------------------------------------------------------------------
# The joint stage's validation (run_sr.py:1131-1138): numpy's MSE and cv2's quarter-size resize
# ------------------------------------------------------------------------------------------------
def numpy_visit_order(shape, strides_a, strides_b):
    """The axes of ``a - b`` (``[H, W, 3]`` operands with these element strides) from the outermost to the innermost
    in the order numpy visits the difference's elements: numpy allocates the difference in 'K' order
    (``npyiter_find_best_axis_ordering``: a stable insertion sort from the innermost axis by stride, where an axis
    moves inward only if every operand with non-zero strides on both axes agrees, C order otherwise), and the mean
    then reduces it in its memory order.  A size-1 axis has stride 0 there."""
    nd = len(shape)
    st = [[0 if shape[ax] == 1 else abs(int(s[ax])) for s in (strides_a, strides_b)] for ax in range(nd)]
    perm = list(range(nd))                        # iterator axes, innermost first: axis j is array axis nd - 1 - j
    for i0 in range(1, nd):
        j0, ipos = perm[i0], i0
        s0 = st[nd - 1 - j0]
        for i1 in range(i0 - 1, -1, -1):
            s1 = st[nd - 1 - perm[i1]]
            ambig, swap = True, False
            for op in range(2):
                if s0[op] != 0 and s1[op] != 0:
                    if s1[op] <= s0[op]:
                        swap = False
                    elif ambig:
                        swap = True
                    ambig = False
            if not ambig:
                if swap:
                    ipos = i1
                else:
                    break
        if ipos != i0:
            perm[ipos + 1:i0 + 1] = perm[ipos:i0]
            perm[ipos] = j0
    return [nd - 1 - j for j in reversed(perm)]


def _cuda_rgb_pair(a, b, what):
    if not (_is_cuda(a) and _is_cuda(b) and a.device == b.device):
        raise RuntimeError(f'{what}: both images must be CUDA tensors on one device, or both numpy arrays')
    if a.dtype != torch.float32 or b.dtype != torch.float32:
        raise TypeError(f'{what}: float32 images expected, got {a.dtype} and {b.dtype}')
    if a.ndim != 3 or a.shape[-1] != 3 or a.shape != b.shape:
        raise ValueError(f'{what}: two [H, W, 3] images of one shape expected, got {tuple(a.shape)} and {tuple(b.shape)}')
    return a.detach(), b.detach()


def rgb_mse(a, b):
    """``np.mean(np.square(a - b))`` of two float32 ``[H, W, 3]`` images (run_sr.py:1132), as ``np.float32``; the PSNR
    is ``-10. * np.log10(rgb_mse(a, b))`` (float32, as the reference's ``sr_psnr``).

    CUDA tensors (both on one device, any strides, e.g. ``sr.permute(1, 2, 0)`` of a ``[3, H, W]`` frame) are scored
    by ``k4_op_mse_f32`` with numpy's result bit for bit: the differences and squares in float32, numpy's pairwise sum
    over the elements in the order numpy would visit arrays of those strides (:func:`numpy_visit_order`), and numpy's
    division; one 4-byte read.  Numpy arrays and CPU tensors are numpy's own expression."""
    if _is_cuda(a) or _is_cuda(b):
        import ctypes as C
        from . import _lib
        a, b = _cuda_rgb_pair(a, b, 'rgb_mse')
        H, W = a.shape[0], a.shape[1]
        dev = a.device
        with torch.cuda.device(dev):
            ws = torch.empty(max(_lib.lib.k4_op_mse_f32_workspace_bytes(H, W), 4), dtype=torch.uint8, device=dev)
            out = torch.empty((), dtype=torch.float32, device=dev)
            order = (C.c_int32 * 3)(*numpy_visit_order(a.shape, a.stride(), b.stride()))
            _cuda_call('k4_op_mse_f32', C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), H, W, _strides3(a), _strides3(b),
                       order, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                       C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        return np.float32(out.item())
    return np.mean(np.square(np.asarray(a) - np.asarray(b)))


def resize_quarter_size(H, W):
    """cv2's ``dsize`` for ``fx = fy = 1/4``: ``(cvRound(H / 4), cvRound(W / 4))``, halves rounded to even."""
    return int(np.rint(H * 0.25)), int(np.rint(W * 0.25))


def _resize_quarter_axis(n, d, clamp_last):
    """Source pairs and weights of the ``d`` outputs along an axis of ``n`` pixels (see :func:`resize_quarter`)."""
    k = np.arange(d)
    inside = 4 * k + 3 <= n
    i0 = np.where(inside, 4 * k + 1, n - 1 if clamp_last else n - 2)
    i1 = np.where(inside, 4 * k + 2, n - 1)
    t = np.where(inside, 0.5, 0.0 if clamp_last else 1.0).astype(np.float32)
    return i0, i1, t


def _lerp_f32(a, b, t):
    """``a + (b - a) t`` in float32, one rounding per operation; ``t == 0`` is ``a`` itself."""
    return np.where(t == 0, a, (a + (b - a) * t).astype(np.float32))


def _resize_quarter_np(x):
    x = np.asarray(x)
    H, W = x.shape[0], x.shape[1]
    h, w = resize_quarter_size(H, W)
    rows_first = H == 3 or W == 3
    y0, y1, ty = _resize_quarter_axis(H, h, rows_first)
    x0, x1, tx = _resize_quarter_axis(W, w, rows_first)
    ty, tx = ty[:, None, None], tx[None, :, None]
    g = lambda ys, xs: x[ys][:, xs]
    if rows_first:
        return _lerp_f32(_lerp_f32(g(y0, x0), g(y1, x0), ty), _lerp_f32(g(y0, x1), g(y1, x1), ty), tx)
    return _lerp_f32(_lerp_f32(g(y0, x0), g(y0, x1), tx), _lerp_f32(g(y1, x0), g(y1, x1), tx), ty)


def resize_quarter(x):
    """``cv2.resize(x, None, fx=1/4, fy=1/4)`` (INTER_LINEAR) of a float32 ``[H, W, 3]`` image, bit for bit with cv2
    4.13's IPP build: the frames run_sr.py:1136 scores LPIPS on when ``load_sr == 1``.  The output is ``[h, w, 3]``
    (:func:`resize_quarter_size`; H and W at least 3).  Along an axis of n pixels output k is ``a + (b - a) t`` of
    pixels 4k+1 and 4k+2 with t = 0.5, or of pixels n-2 and n-1 with t = 1 when 4k + 3 > n; columns first, then rows.
    With H or W equal to 3 cv2 goes rows first and reads pixel n-1 alone past the edge.

    CUDA tensors (any strides, e.g. ``sr.permute(1, 2, 0)``) run on the GPU (``k4_op_resize_quarter``) and give a
    contiguous CUDA tensor; numpy arrays and CPU tensors take the numpy restatement and give a numpy array."""
    if not (x.ndim == 3 and x.shape[-1] == 3 and x.dtype in (np.float32, torch.float32)):
        raise ValueError(f'resize_quarter: a float32 [H, W, 3] image expected, got {x.dtype} {tuple(x.shape)}')
    H, W = x.shape[0], x.shape[1]
    if H < 3 or W < 3:
        raise ValueError(f'resize_quarter: {H} x {W} has no pixels at a quarter of its size (cv2 rejects it too)')
    if not _is_cuda(x):
        return _resize_quarter_np(x)
    import ctypes as C
    x = x.detach()
    out = torch.empty((*resize_quarter_size(H, W), 3), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _cuda_call('k4_op_resize_quarter', C.c_void_p(x.data_ptr()), H, W, _strides3(x), C.c_void_p(out.data_ptr()),
                   C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
    return out


# ------------------------------------------------------------------------------------------------
# LPIPS (lib/utils.py:137-149)
# ------------------------------------------------------------------------------------------------
_LPIPS_NETS = {'vgg': 0, 'alex': 1}                                 # K4_LPIPS_VGG / K4_LPIPS_ALEX
_LPIPS_CONVS = {
    'vgg': ['net.slice1.0', 'net.slice1.2', 'net.slice2.5', 'net.slice2.7', 'net.slice3.10', 'net.slice3.12',
            'net.slice3.14', 'net.slice4.17', 'net.slice4.19', 'net.slice4.21', 'net.slice5.24', 'net.slice5.26',
            'net.slice5.28'],
    'alex': ['net.slice1.0', 'net.slice2.3', 'net.slice3.6', 'net.slice4.8', 'net.slice5.10'],
}
_LPIPS_SHIFT, _LPIPS_SCALE = (-.030, -.088, -.188), (.458, .448, .450)
__LPIPS__ = {}


def _lpips_state_dict(net_name):
    """The pretrained weights, as the reference's init_lpips builds its module (needs the ``lpips`` package)."""
    import lpips
    print(f'init_lpips: lpips_{net_name}')
    return lpips.LPIPS(net=net_name, version='0.1').state_dict()


class LpipsNet:
    """``lpips.LPIPS(net=net_name, version='0.1')`` on one CUDA device (``k4_lpips_create``, csrc/k4_lpips.cu) from a
    state dict with its keys (``net.slice*``, ``lin0..4.model.1.weight``; a ``scaling_layer`` must hold lpips' own
    constants)."""

    def __init__(self, net_name, state_dict, device):
        import ctypes as C
        from . import _lib
        if net_name not in _LPIPS_NETS:
            raise ValueError(f"rgb_lpips: net_name must be 'vgg' or 'alex', got {net_name!r}")
        for k, ref in (('scaling_layer.shift', _LPIPS_SHIFT), ('scaling_layer.scale', _LPIPS_SCALE)):
            if k in state_dict and not torch.equal(state_dict[k].detach().float().cpu().view(-1), torch.tensor(ref)):
                raise ValueError(f'rgb_lpips: {k} differs from lpips 0.1\'s constants {ref}')
        keys = [k + s for k in _LPIPS_CONVS[net_name] for s in ('.weight', '.bias')] + [f'lin{i}.model.1.weight' for i in range(5)]
        missing = [k for k in keys if k not in state_dict]
        if missing:
            raise KeyError(f'rgb_lpips: the state dict lacks {missing}')
        self.net_name, self.device, self._lib, self.handle = net_name, device, _lib, None
        params = [state_dict[k].detach().to(device=device, dtype=torch.float32).contiguous() for k in keys]
        ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
        h = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(_lib.lib.k4_lpips_create(_LPIPS_NETS[net_name], ptrs, len(params),
                                                C.c_void_p(torch.cuda.current_stream(device).cuda_stream), C.byref(h)),
                       'k4_lpips_create')
        self.handle = h

    def __del__(self):
        if getattr(self, 'handle', None) is not None:
            self._lib.lib.k4_lpips_destroy(self.handle)
            self.handle = None

    def __call__(self, img0, img1):
        """The score of two ``[H, W, 3]`` float32 CUDA images on this device (any strides) as a Python float."""
        import ctypes as C
        H, W = img0.shape[0], img0.shape[1]
        with torch.cuda.device(self.device):
            ws = torch.empty(self._lib.lib.k4_lpips_workspace_bytes(self.handle, H, W), dtype=torch.uint8, device=self.device)
            if ws.numel() == 0:
                raise ValueError(f'rgb_lpips: {H} x {W} is outside what lpips {self.net_name} takes '
                                 f'({"16" if self.net_name == "vgg" else "31"} .. 16384 pixels per side)')
            out = torch.empty((), dtype=torch.float64, device=self.device)
            self._lib.check(self._lib.lib.k4_lpips_forward(
                self.handle, C.c_void_p(img0.data_ptr()), C.c_void_p(img1.data_ptr()), _strides3(img0), _strides3(img1),
                H, W, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)), 'k4_lpips_forward')
        return float(out.item())


def rgb_lpips(np_gt, np_im, net_name, device=None, weights=None):
    """LPIPS 0.1 of two ``[H, W, 3]`` images in [0, 1] as ``lib/utils.py:144-149`` computes it
    (``lpips.LPIPS(net=net_name, version='0.1')(gt, im, normalize=True).item()``), on the GPU (csrc/k4_lpips.cu):
    VGG16's convolutions on the decoder's wgmma kernels with every value an fp16 pair hi + lo (fp32-class), AlexNet's
    in fp32, the head in fp64.  The score is a float, bitwise reproducible.

    ``np_gt``, ``np_im``: numpy arrays, or tensors of any strides (e.g. ``sr.permute(1, 2, 0)`` of a ``[3, H, W]`` 4K
    frame, scored in place when it is float32 on the GPU).  ``device``: where to score; CUDA tensors are scored on
    their own device.  ``weights``: a state dict with ``lpips.LPIPS``' keys; by default the pretrained weights of the
    ``lpips`` package, loaded once per net and device (without the package this raises ``ImportError``, as the
    reference does)."""
    cuda_in = [t for t in (np_gt, np_im) if _is_cuda(t)]
    dev = cuda_in[0].device if cuda_in else torch.device(device if device is not None else 'cuda')
    if dev.type != 'cuda':
        raise ValueError(f'rgb_lpips runs on a CUDA device (got {dev})')
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    if weights is None:
        key = (net_name, dev)
        if key not in __LPIPS__:
            __LPIPS__[key] = LpipsNet(net_name, _lpips_state_dict(net_name), dev)
        net = __LPIPS__[key]
    else:
        net = LpipsNet(net_name, weights, dev)

    def as_image(x):
        x = torch.from_numpy(np.asarray(x)) if not isinstance(x, torch.Tensor) else x.detach()
        if x.ndim != 3 or x.shape[-1] != 3:
            raise ValueError(f'rgb_lpips: [H, W, 3] images expected, got shape {tuple(x.shape)}')
        return x.to(device=dev, dtype=torch.float32)

    img0, img1 = as_image(np_gt), as_image(np_im)
    if img0.shape != img1.shape:
        raise ValueError(f'rgb_lpips: the images differ in shape: {tuple(img0.shape)} and {tuple(img1.shape)}')
    return net(img0, img1)


# ------------------------------------------------------------------------------------------------
# The depth video of run_sr.py --render_video (run_sr.py:1459-1463)
# ------------------------------------------------------------------------------------------------
def rainbow_lut_u8():
    """``to8b`` of matplotlib's ``rainbow`` colormap table, ``[256, 3]`` uint8.  matplotlib defines ``rainbow`` as a
    ``LinearSegmentedColormap`` of N = 256 entries sampled at ``np.linspace(0, 1, 256)`` from red ``|2x - 0.5|``, green
    ``sin(pi x)`` and blue ``cos(pi x / 2)``, each clipped to [0, 1]; the expressions below are its own."""
    x = np.linspace(0, 1, 256)
    lut = np.clip(np.stack([np.abs(2 * x - 0.5), np.sin(x * np.pi), np.cos(x * np.pi / 2)], -1), 0, 1)
    return to8b(lut)


def _f32_keys(v):
    """Order-preserving uint32 keys of float32 values (-0.0 before +0.0, every NaN last)."""
    u = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32)
    k = np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)
    k[np.isnan(v)] = 0xffffffff
    return k


def _f32_of_keys(k):
    return np.where(k & 0x80000000, k & 0x7fffffff, ~k).astype(np.uint32).view(np.float32)


def _quantile_fractions(q):
    """``q / 100`` exactly as ``np.percentile`` computes it for float32 data, for a pair of percentiles."""
    qf = np.true_divide(np.asarray(q, dtype=np.float64), np.float32(100))
    if qf.shape != (2,):
        raise ValueError(f'q must be a pair of percentiles, got {q!r}')
    if not (np.all(0 <= qf) and np.all(qf <= 1)):
        raise ValueError('Percentiles must be in the range [0, 100]')
    return qf


def masked_quantiles_np(values, q=(5, 95)):
    """``np.percentile(values, q)`` (method 'linear') of float32 values, restated from their order statistics as the
    kernel computes it: sorted order-preserving keys, numpy's indexes (``_get_indexes``: virtual index ``(n - 1) q``,
    both neighbours the last value at or above the last index, where numpy's previous index is -1 and its gamma
    ``virtual + 1``) and numpy's ``_lerp`` (the difference in float32, the rest in float64).  Returns two
    ``np.float64``; NaN among the values gives NaN, as numpy; no values raise ``ValueError``."""
    qf = _quantile_fractions(q)
    v = np.asarray(values, dtype=np.float32).ravel()
    n = v.size
    if n == 0:
        raise ValueError('the depth video needs at least one pixel with bgmap < 0.1')
    s = _f32_of_keys(np.sort(_f32_keys(v)))
    out = []
    for t in qf:
        prev, nxt, gamma = _np_indexes(n, t)
        r = _np_lerp(s[prev], s[nxt], gamma)
        out.append(np.float64(np.nan) if np.isnan(v).any() else np.float64(r))
    return out[0], out[1]


def _np_indexes(n, t):
    """numpy's 'linear' order statistics of quantile fraction ``t`` among ``n`` values: ``(prev, next, gamma)``."""
    vi = np.float64(n - 1) * t
    if vi >= n - 1:
        return n - 1, n - 1, vi - np.float64(-1)
    prev = int(np.floor(vi))
    return prev, prev + 1, vi - np.float64(prev)


def _np_lerp(a, b, gamma):
    """numpy's ``_lerp`` of two float32 order statistics: the difference in float32, the rest in float64."""
    with np.errstate(invalid='ignore'):                                     # inf - inf, as numpy's own
        d = np.float64(np.float32(b - a))
        return np.float64(b) - d * (1 - gamma) if gamma >= 0.5 else np.float64(a) + d * gamma


# The split select of k4_op_masked_quantiles_hist / _select restated: one share's int64 histogram per pass, and the
# select of a summed histogram.  ``state`` is the per-pass state the C workspace holds (a dict, empty before pass 0).
MQ_BINS, MQ_RANKS = 2048, 4
MQ_HIST_LEN = MQ_RANKS * MQ_BINS + 2                  # include/k4nerf.h's K4_MASKED_QUANTILES_HIST_LEN
_MQ_SHIFT, _MQ_NBINS = (21, 10, 0), (2048, 2048, 1024)


def masked_quantiles_hist_np(p, values, state):
    """Pass ``p``'s histogram of one share's selected float32 ``values`` (``depths_vis[bgmaps < 0.1]``), int64
    ``[MQ_HIST_LEN]``: pass 0 the top 11 bits of every key, the count and the NaN count; passes 1 and 2 the next digit of
    the keys under each distinct rank prefix, in the slot of the first rank with that prefix."""
    v = np.asarray(values, dtype=np.float32).ravel()
    k = _f32_keys(v).astype(np.int64)
    hist = np.zeros(MQ_HIST_LEN, np.int64)
    nb = _MQ_NBINS[p]
    if p == 0:
        hist[:nb] = np.bincount(k >> _MQ_SHIFT[0], minlength=nb)
        hist[-2], hist[-1] = k.size, np.count_nonzero(np.isnan(v))
        return hist
    for r in range(MQ_RANKS):
        if state['slot'][r] == r:
            under = k[(k >> _MQ_SHIFT[p - 1]) == state['prefix'][r]]
            hist[r * MQ_BINS:r * MQ_BINS + nb] = np.bincount((under >> _MQ_SHIFT[p]) & (nb - 1), minlength=nb)
    return hist


def masked_quantiles_select_np(p, hist, q, state):
    """Pass ``p``'s select on the summed ``hist``: pass 0 turns the count into numpy's indexes, every pass narrows each
    of the four ranks (prev / next of both quantiles) to one more digit, pass 2 returns ``(dmin, dmax, count)`` as
    ``k4_op_masked_quantiles`` writes them (NaN quantiles for no or NaN values)."""
    hist = np.asarray(hist, dtype=np.int64)
    if p == 0:
        n = int(hist[-2])
        state.update(count=n, nans=int(hist[-1]), prefix=[0] * MQ_RANKS, slot=[0] * MQ_RANKS, rank=[], gamma=[])
        for t in _quantile_fractions(q):
            prev, nxt, gamma = _np_indexes(n, t) if n else (0, 0, 0.0)
            state['rank'] += [prev, nxt]
            state['gamma'].append(gamma)
    nb = _MQ_NBINS[p]
    for r in range(MQ_RANKS):
        slot = state['slot'][r]
        c = np.cumsum(hist[slot * MQ_BINS:slot * MQ_BINS + nb])
        b = int(np.searchsorted(c, state['rank'][r], side='right'))           # the first bin whose prefix sum passes it
        if b == nb:                                                           # no values at all: as the kernel, the last
            b, below = nb - 1, state['rank'][r]
        else:
            below = int(c[b - 1]) if b else 0
        state['prefix'][r] = (state['prefix'][r] << (10 if p == 2 else 11)) | b
        state['rank'][r] -= below
    state['slot'] = [state['prefix'].index(x) for x in state['prefix']]
    if p < 2:
        return None
    n, v = state['count'], _f32_of_keys(np.array(state['prefix'], np.uint32))
    out = [np.float64(np.nan) if n == 0 or state['nans'] else np.float64(_np_lerp(v[2 * j], v[2 * j + 1], state['gamma'][j]))
           for j in range(2)]
    return out[0], out[1], n


def _flip_rot(frames, render_video_flipy, render_video_rot90):
    """``render_video_flipy`` then ``render_video_rot90`` of render.py's ``_post``, on ``[n, H, W, ...]`` frames."""
    if render_video_flipy:
        frames = np.flip(frames, axis=1)
    return np.ascontiguousarray(np.rot90(frames, k=render_video_rot90, axes=(1, 2)))


def _frames_of(x, name):
    """``[n, H, W]`` of an ``[n, H, W]`` or ``[n, H, W, 1]`` array / tensor (a view)."""
    if x.ndim == 4 and x.shape[-1] == 1:
        x = x[..., 0]
    if x.ndim != 3:
        raise ValueError(f'{name} must be [n, H, W] or [n, H, W, 1], got shape {tuple(x.shape)}')
    return x


def _depth_video_np(depths, bgmaps, q, render_video_flipy, render_video_rot90):
    """run_sr.py:1459-1463 in numpy, the colormap restated (``rainbow_lut_u8``) and the percentiles by
    ``masked_quantiles_np``; ``Colormap.__call__``'s index: trunc(256 x), 256 -> 255, NaN -> the 'bad' colour."""
    depths = _frames_of(np.asarray(depths, dtype=np.float32), 'depths')
    bgmaps = _frames_of(np.asarray(bgmaps, dtype=np.float32), 'bgmaps')
    if depths.shape != bgmaps.shape:
        raise ValueError(f'depths {depths.shape} and bgmaps {bgmaps.shape} differ')
    depths_vis = depths * (1 - bgmaps) + bgmaps
    dmin, dmax = masked_quantiles_np(depths_vis[bgmaps < 0.1], q)
    return _colour_np(depths_vis, dmin, dmax, render_video_flipy, render_video_rot90), dmin, dmax


def _colour_np(depths_vis, dmin, dmax, render_video_flipy, render_video_rot90):
    """The rainbow frames of ``depths_vis`` under the range ``dmin, dmax`` (run_sr.py:1461-1463), flipped and rotated."""
    with np.errstate(divide='ignore', invalid='ignore'):
        x = 1 - np.clip((depths_vis - dmin) / (dmax - dmin), 0, 1)
        xa = x * 256
        xa[xa == 256] = 255
        bad = np.isnan(xa)
        idx = xa.astype(int)
    idx[bad] = 0
    frames = rainbow_lut_u8()[idx]
    frames[bad] = 0
    return _flip_rot(frames, render_video_flipy, render_video_rot90)


def _strides3(t):
    import ctypes as C
    return (C.c_int64 * 3)(*t.stride())


def _cuda_call(fn, *args):
    from . import _lib
    _lib.check(getattr(_lib.lib, fn)(*args), fn)


def _depth_video_cuda(depths, bgmaps, q, render_video_flipy, render_video_rot90):
    """``k4_op_masked_quantiles`` + ``k4_op_depth_video_u8`` (csrc/k4_video.cu) on float32 CUDA tensors, read in place;
    one 24-byte read of the range and count between them."""
    import ctypes as C
    from . import _lib
    depths, bgmaps = _cuda_frames(depths, bgmaps)
    n, H, W = depths.shape
    qf = _quantile_fractions(q)
    k = int(render_video_rot90) % 4
    dev = depths.device
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        ws = torch.empty(_lib.lib.k4_op_masked_quantiles_workspace_bytes(n, H, W), dtype=torch.uint8, device=dev)
        res = torch.empty(3, dtype=torch.int64, device=dev)              # dmin, dmax (fp64 bits), count
        sd, sb = _strides3(depths), _strides3(bgmaps)
        _cuda_call('k4_op_masked_quantiles', C.c_void_p(depths.data_ptr()), C.c_void_p(bgmaps.data_ptr()), n, H, W, sd, sb,
                   (C.c_double * 2)(*qf.tolist()), C.c_void_p(res.data_ptr()), C.c_void_p(res.data_ptr() + 16),
                   C.c_void_p(ws.data_ptr()), ws.numel(), stream)
        host = res.cpu().numpy()
        if host[2] == 0:
            raise ValueError('the depth video needs at least one pixel with bgmap < 0.1')
        dmin, dmax = host[:2].view(np.float64)
        out = _colour_cuda(depths, bgmaps, res, render_video_flipy, k, stream)
    return out, np.float64(dmin), np.float64(dmax)


def _cuda_frames(depths, bgmaps):
    """The checked ``[n, H, W]`` float32 views of CUDA ``depths`` / ``bgmaps`` on one device."""
    if not (_is_cuda(depths) and _is_cuda(bgmaps) and depths.device == bgmaps.device):
        raise RuntimeError('depth_video_frames: depths and bgmaps must both be numpy / CPU or both on one CUDA device')
    if depths.dtype != torch.float32 or bgmaps.dtype != torch.float32:
        raise TypeError(f'depth_video_frames: float32 depths and bgmaps expected, got {depths.dtype} and {bgmaps.dtype}')
    depths, bgmaps = _frames_of(depths.detach(), 'depths'), _frames_of(bgmaps.detach(), 'bgmaps')
    if depths.shape != bgmaps.shape:
        raise ValueError(f'depths {tuple(depths.shape)} and bgmaps {tuple(bgmaps.shape)} differ')
    return depths, bgmaps


def _colour_cuda(depths, bgmaps, res, render_video_flipy, k, stream):
    """``k4_op_depth_video_u8`` of ``[n, H, W]`` CUDA frames under the device range ``res[:2]`` (fp64 bits)."""
    import ctypes as C
    n, H, W = depths.shape
    out = torch.empty((n, W, H, 3) if k & 1 else (n, H, W, 3), dtype=torch.uint8, device=depths.device)
    if n == 0:
        return out
    lut = np.ascontiguousarray(rainbow_lut_u8())
    _cuda_call('k4_op_depth_video_u8', C.c_void_p(depths.data_ptr()), C.c_void_p(bgmaps.data_ptr()), n, H, W,
               _strides3(depths), _strides3(bgmaps), C.c_void_p(res.data_ptr()), lut.ctypes.data_as(C.POINTER(C.c_uint8)),
               int(bool(render_video_flipy)), k, C.c_void_p(out.data_ptr()), stream)
    return out


def depth_video_frames(depths, bgmaps, q=(5, 95), render_video_flipy=False, render_video_rot90=0, return_range=False):
    """The depth video of run_sr.py --render_video (run_sr.py:1459-1463) as uint8 frames ``[n, H', W', 3]``:
    ``depths_vis = depths * (1 - bgmaps) + bgmaps`` (float32), ``dmin, dmax = np.percentile(depths_vis[bgmaps < 0.1],
    q)``, then ``to8b`` of matplotlib's ``rainbow`` colormap of ``1 - clip((depths_vis - dmin) / (dmax - dmin), 0, 1)``,
    flipped (``render_video_flipy``, axis 0 of a frame) and then rotated (``np.rot90`` by ``render_video_rot90``) as
    ``render_viewpoints`` flips and rotates its outputs.  H' x W' is W x H for an odd rotation.

    ``depths``, ``bgmaps``: ``[n, H, W, 1]`` (as ``render_viewpoints`` returns them) or ``[n, H, W]``, float32.  CUDA
    tensors run on the GPU (``k4_op_masked_quantiles`` and ``k4_op_depth_video_u8``, any strides) and give a CUDA
    tensor; numpy arrays and CPU tensors take the numpy restatement and give a numpy array.  Both give numpy's values
    bit for bit.  ``return_range=True`` also returns ``(dmin, dmax)`` as ``np.float64``.

    Edge cases, all as numpy and matplotlib: with ``dmax == dmin`` a pixel below the range is colour 255 (x = 1),
    above it colour 0, and on it 0 / 0 = NaN, the colormap's 'bad' colour (0, 0, 0); pixels on dmin / dmax map to
    x = 1 / 0; ``bgmaps == 0.1`` is not selected; NaN depths give the bad colour, and a NaN among the selected values
    makes the range NaN.  No selected pixel raises ``ValueError`` (numpy raises ``IndexError`` there).  The reference's
    ``.squeeze()`` would also drop a frame axis of length 1; here the shape stays ``[n, H', W', 3]``."""
    if _is_cuda(depths) or _is_cuda(bgmaps):
        out, dmin, dmax = _depth_video_cuda(depths, bgmaps, q, render_video_flipy, render_video_rot90)
    else:
        out, dmin, dmax = _depth_video_np(depths, bgmaps, q, render_video_flipy, render_video_rot90)
    return (out, (dmin, dmax)) if return_range else out


def _depth_video_sharded_cuda(depths, bgmaps, q, render_video_flipy, k, all_reduce):
    """The split passes (``k4_op_masked_quantiles_hist`` / ``_select``) with ``all_reduce`` summing each pass's
    histogram over the shares, then ``k4_op_depth_video_u8`` of this share's frames; one 24-byte read of the range."""
    import ctypes as C
    from . import _lib
    depths, bgmaps = _cuda_frames(depths, bgmaps)
    n, H, W = depths.shape
    dev = depths.device
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        ws = torch.empty(_lib.lib.k4_op_masked_quantiles_pass_workspace_bytes(), dtype=torch.uint8, device=dev)
        hist = torch.empty(_lib.K4_MASKED_QUANTILES_HIST_LEN, dtype=torch.int64, device=dev)
        res = torch.empty(3, dtype=torch.int64, device=dev)              # dmin, dmax (fp64 bits), count
        sd, sb, q = _strides3(depths), _strides3(bgmaps), (C.c_double * 2)(*_quantile_fractions(q).tolist())
        for p in range(3):
            hist.zero_()
            _cuda_call('k4_op_masked_quantiles_hist', p, C.c_void_p(depths.data_ptr()), C.c_void_p(bgmaps.data_ptr()),
                       n, H, W, sd, sb, C.c_void_p(hist.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), stream)
            all_reduce(hist)
            _cuda_call('k4_op_masked_quantiles_select', p, C.c_void_p(hist.data_ptr()), q, C.c_void_p(res.data_ptr()),
                       C.c_void_p(res.data_ptr() + 16), C.c_void_p(ws.data_ptr()), ws.numel(), stream)
        host = res.cpu().numpy()
        if host[2] == 0:
            raise ValueError('the depth video needs at least one pixel with bgmap < 0.1')
        dmin, dmax = host[:2].view(np.float64)
        out = _colour_cuda(depths, bgmaps, res, render_video_flipy, k, stream)
    return out, np.float64(dmin), np.float64(dmax)


def _depth_video_sharded_np(depths, bgmaps, q, render_video_flipy, k, all_reduce):
    """The numpy restatement of the split passes (``masked_quantiles_hist_np`` / ``_select_np``), then the colours."""
    depths = _frames_of(np.asarray(depths, dtype=np.float32), 'depths')
    bgmaps = _frames_of(np.asarray(bgmaps, dtype=np.float32), 'bgmaps')
    if depths.shape != bgmaps.shape:
        raise ValueError(f'depths {depths.shape} and bgmaps {bgmaps.shape} differ')
    depths_vis = depths * (1 - bgmaps) + bgmaps
    values, state = depths_vis[bgmaps < 0.1], {}
    for p in range(3):
        hist = torch.from_numpy(masked_quantiles_hist_np(p, values, state))
        all_reduce(hist)
        res = masked_quantiles_select_np(p, hist.numpy(), q, state)
    dmin, dmax, count = res
    if count == 0:
        raise ValueError('the depth video needs at least one pixel with bgmap < 0.1')
    return _colour_np(depths_vis, dmin, dmax, render_video_flipy, k), dmin, dmax


def depth_video_frames_sharded(depths, bgmaps, q=(5, 95), render_video_flipy=False, render_video_rot90=0, group=None,
                               return_range=False):
    """:func:`depth_video_frames` of a video whose frames are spread over the ranks of ``group``: each rank passes its
    own ``[n_r, H, W]`` (or ``[n_r, H, W, 1]``) depth and bgmap frames, ``n_r`` may be 0, and gets its own frames'
    colours, ``[n_r, H', W', 3]`` uint8, under the range of ALL the ranks' frames.  That range is exact: each of the
    select's three passes builds the integer histogram of the rank's own keys (``k4_op_masked_quantiles_hist``), one
    ``all_reduce(SUM)`` adds them, and every rank selects on the sum (``k4_op_masked_quantiles_select``), so all ranks
    reach the same order statistics as ``np.percentile`` over every frame, bit for bit.  CUDA tensors run on the GPU
    (a gloo group takes the histogram through the host); numpy arrays and CPU tensors take the numpy restatement and
    give numpy arrays.  On a group of one rank (or without a process group) the result is :func:`depth_video_frames`'.
    No selected pixel on any rank raises ``ValueError`` on every rank.  Collective: every rank of ``group`` calls it."""
    from . import dist as kdist
    _quantile_fractions(q)                                  # a bad q raises before any collective
    k = int(render_video_rot90) % 4
    all_reduce = lambda t: kdist.all_reduce_sum(t, group)
    if _is_cuda(depths) or _is_cuda(bgmaps):
        out, dmin, dmax = _depth_video_sharded_cuda(depths, bgmaps, q, render_video_flipy, k, all_reduce)
    else:
        out, dmin, dmax = _depth_video_sharded_np(depths, bgmaps, q, render_video_flipy, k, all_reduce)
    return (out, (dmin, dmax)) if return_range else out


def frame_u8_cuda(rgb, render_video_flipy=False, render_video_rot90=0, out=None):
    """``to8b`` of one float32 ``[H, W, 3]`` CUDA frame (any strides, e.g. ``sr.permute(1, 2, 0)`` of a decoder
    output), flipped and rotated like :func:`depth_video_frames`, by ``k4_op_frame_u8``: a uint8 ``[H', W', 3]`` CUDA
    tensor (written into ``out`` when given, which must be contiguous)."""
    import ctypes as C
    if not _is_cuda(rgb) or rgb.dtype != torch.float32 or rgb.ndim != 3 or rgb.shape[-1] != 3:
        raise ValueError(f'frame_u8_cuda: a float32 [H, W, 3] CUDA tensor expected, got {getattr(rgb, "shape", None)}')
    H, W = rgb.shape[0], rgb.shape[1]
    k = int(render_video_rot90) % 4
    shape = (W, H, 3) if k & 1 else (H, W, 3)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=rgb.device)
    elif tuple(out.shape) != shape or out.dtype != torch.uint8 or not out.is_contiguous() or out.device != rgb.device:
        raise ValueError(f'frame_u8_cuda: out must be a contiguous uint8 {shape} tensor on {rgb.device}')
    rgb = rgb.detach()
    with torch.cuda.device(rgb.device):
        _cuda_call('k4_op_frame_u8', C.c_void_p(rgb.data_ptr()), H, W, _strides3(rgb), int(bool(render_video_flipy)), k,
                   C.c_void_p(out.data_ptr()), C.c_void_p(torch.cuda.current_stream(rgb.device).cuda_stream))
    return out


# ------------------------------------------------------------------------------------------------
# PNG files of uint8 frames (run.py:165, run_sr.py:175 / 1396: imageio.imwrite)
# ------------------------------------------------------------------------------------------------
def png_encode(frame):
    """The PNG file of a contiguous uint8 ``[H, W, 3]`` CUDA frame, encoded on its device by ``k4_png_encode``
    (csrc/k4_png.cu), as ``bytes``.  The encode is queued on the current stream; the only host synchronisations are
    the copy of the file's length and then of its bytes."""
    import ctypes as C
    from . import _lib
    if not (_is_cuda(frame) and frame.dtype == torch.uint8 and frame.ndim == 3 and frame.shape[-1] == 3):
        raise ValueError(f'png_encode: a uint8 [H, W, 3] CUDA tensor expected, got {getattr(frame, "dtype", type(frame))} '
                         f'{tuple(getattr(frame, "shape", ()))}')
    frame = frame.detach().contiguous()
    H, W = frame.shape[0], frame.shape[1]
    dev = frame.device
    bound = _lib.lib.k4_png_encode_bound(H, W)
    if bound == 0:
        raise ValueError(f'png_encode: a {H} x {W} frame does not fit one PNG IDAT chunk')
    with torch.cuda.device(dev):
        ws = torch.empty(_lib.lib.k4_png_workspace_bytes(H, W), dtype=torch.uint8, device=dev)
        out = torch.empty(bound, dtype=torch.uint8, device=dev)
        n = torch.empty((), dtype=torch.int64, device=dev)
        _cuda_call('k4_png_encode', C.c_void_p(frame.data_ptr()), H, W, C.c_void_p(out.data_ptr()), bound,
                   C.c_void_p(n.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                   C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        return out[:int(n.item())].cpu().numpy().tobytes()


def write_png(filename, frame):
    """Write ``frame`` as the PNG file ``filename``: a uint8 ``[H, W, 3]`` CUDA tensor is encoded on its device
    (:func:`png_encode`), a numpy array goes through the host writer ``render_viewpoints``' dumps use
    (``render._write_png``: imageio, PIL or cv2).  Anything else raises ``TypeError``."""
    if _is_cuda(frame):
        data = png_encode(frame)
        with open(filename, 'wb') as f:
            f.write(data)
    elif isinstance(frame, np.ndarray):
        from .render import _write_png
        _write_png(filename, frame)
    else:
        raise TypeError(f'write_png: a CUDA tensor or a numpy array expected, got {type(frame).__name__}')
