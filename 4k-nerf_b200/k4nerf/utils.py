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
