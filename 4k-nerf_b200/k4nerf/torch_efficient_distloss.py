"""Drop-in for ``flatten_eff_distloss``, the one name the reference's training loop imports from the third-party
package ``torch_efficient_distloss`` (run_sr.py:16; called at run_sr.py:536-542 and :977-989 whenever
``weight_distortion > 0``, which every LLFF config sets).  Backed by csrc/k4_distloss.cu through the C ABI.

    flatten_eff_distloss(w, m, interval, ray_id)
        = (sum_r sum_{i,j in r} w_i w_j |m_i - m_j| + interval / 3 * sum_i w_i^2) / (ray_id.max() + 1)

for m sorted within each ray; for any m, the loss is 2 sum_i w_i (m_i W<i - WM<i) over exclusive in-ray prefixes plus
the interval term.  w, m: [M] float32 CUDA tensors (w may require grad); ray_id: [M] int64, non-decreasing; interval: a
Python number or a one-element tensor.  Only w receives a gradient.  Rays without samples, trailing ones included, do
not count in the divisor.  Loss and gradient are bitwise reproducible; neither the forward nor the backward
synchronises the host (the divisor stays on the device).  As in ``render_utils_cuda``, non-CUDA, non-contiguous or
wrongly typed inputs raise RuntimeError, and so does an empty list (``ray_id.max()`` of nothing).
"""
import numbers

import torch

from . import _lib
from .render_utils_cuda import _call, _chk, _p, _s


def _check(w, m, ray_id):
    """Types and shapes; the caller checks device and layout (render_utils_cuda._chk) after its own arguments."""
    for t in (w, m, ray_id):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError('distortion loss: w, m and ray_id must be tensors')
    if w.dtype != torch.float32 or m.dtype != torch.float32 or ray_id.dtype != torch.int64:
        raise RuntimeError('distortion loss: w and m must be float32, ray_id int64')
    if w.dim() != 1 or m.shape != w.shape or ray_id.shape != w.shape:
        raise RuntimeError(f'distortion loss: w, m and ray_id must be [M] (got {tuple(w.shape)}, {tuple(m.shape)}, '
                           f'{tuple(ray_id.shape)})')
    if not (w.device == m.device == ray_id.device):
        raise RuntimeError('distortion loss: w, m and ray_id must be on one device')
    if w.numel() == 0:
        raise RuntimeError('distortion loss: empty sample list (ray_id.max() of an empty tensor)')


def _interval(interval, device):
    """(host value, device scalar or None): a CUDA tensor stays on the device (reading it would synchronise)."""
    if isinstance(interval, torch.Tensor):
        if interval.numel() != 1 or not (interval.is_floating_point() or interval.dtype in (torch.int32, torch.int64)):
            raise RuntimeError(f'distortion loss: interval must be a number or a one-element tensor (got {interval.dtype} '
                               f'{tuple(interval.shape)})')
        if not interval.is_cuda:
            return float(interval), None
        if interval.device != device:
            raise RuntimeError('distortion loss: interval must be on the samples\' device')
        return 0.0, interval.detach().reshape(1).to(torch.float32).contiguous()
    if isinstance(interval, bool) or not isinstance(interval, numbers.Real):
        raise RuntimeError(f'distortion loss: interval must be a number or a one-element tensor (got {type(interval).__name__})')
    return float(interval), None


def _ws(n, device):
    return torch.empty(_lib.lib.k4_op_distloss_workspace_bytes(n), dtype=torch.uint8, device=device)


def autograd_forward(ctx, w, m, interval, ray_id, divide_by_n):
    """Forward of a distortion-loss autograd Function: the loss as a 0-dim float32 tensor.  The backward reads the
    workspace the forward filled (the divisor and the per-tile carries), so it is saved with the inputs."""
    _check(w, m, ray_id)
    iv, d_iv = _interval(interval, w.device)
    _chk(w, m, ray_id)
    n = w.numel()
    loss = torch.empty((), dtype=torch.float32, device=w.device)
    ws = _ws(n, w.device)
    _call('k4_op_distloss_forward', _p(w), _p(m), _p(ray_id), n, iv, None if d_iv is None else _p(d_iv), _p(loss),
          _p(ws), ws.numel(), _s(w))
    ctx.iv, ctx.divide_by_n = iv, divide_by_n
    ctx.save_for_backward(w, m, ray_id, ws, *([] if d_iv is None else [d_iv]))
    return loss


def autograd_backward(ctx, grad_loss):
    w, m, ray_id, ws, *d_iv = ctx.saved_tensors
    g = grad_loss.detach().reshape(1).to(device=w.device, dtype=torch.float32).contiguous()
    grad = torch.empty_like(w)
    _call('k4_op_distloss_backward', _p(w), _p(m), _p(ray_id), w.numel(), ctx.iv, _p(d_iv[0]) if d_iv else None, _p(g),
          1 if ctx.divide_by_n else 0, _p(ws), ws.numel(), _p(grad), _s(w))
    return grad, None, None, None


class FlattenEffDistLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, w, m, interval, ray_id):
        return autograd_forward(ctx, w, m, interval, ray_id, divide_by_n=True)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        return autograd_backward(ctx, grad_loss)


def flatten_eff_distloss(w, m, interval, ray_id):
    return FlattenEffDistLoss.apply(w, m, interval, ray_id)


__all__ = ['flatten_eff_distloss']
