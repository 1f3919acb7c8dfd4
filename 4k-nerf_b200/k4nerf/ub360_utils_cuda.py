"""Drop-in for the reference's pybind module ``ub360_utils_cuda`` (lib/cuda/ub360_utils.cpp:20-26), plus the
``segment_cumsum`` that the reference's DistortionLoss (lib/dcvgo.py:390) calls and its extension does not define."""
import torch

from .render_utils_cuda import _call, _chk, _p, _s, cumdist_thres  # noqa: F401
from .torch_efficient_distloss import _check, _ws


def segment_cumsum(w, s, ray_id):
    """Per-ray sums of w and w * s over a flat sample list (w, s [M] float32, ray_id [M] int64 non-decreasing):
    returns ``[w_prefix [M], w_total [n], ws_prefix [M], ws_total [n]]`` with n = ray_id.max() + 1, the prefixes
    exclusive (the sum over the earlier samples of the sample's ray) and a ray without samples totalling 0.  Sizing
    the totals needs n on the host: the call's one synchronisation (``ray_id.max()``), as ``sample_pts_on_rays``
    reads its point count."""
    _check(w, s, ray_id)
    _chk(w, s, ray_id)
    n = int(ray_id.max()) + 1
    if n < 1:
        raise RuntimeError('segment_cumsum: ray ids must be >= 0')
    M = w.numel()
    w_prefix, ws_prefix = torch.empty_like(w), torch.empty_like(w)
    w_total = torch.empty(n, dtype=torch.float32, device=w.device)
    ws_total = torch.empty(n, dtype=torch.float32, device=w.device)
    ws = _ws(M, w.device)
    _call('k4_op_segment_cumsum', _p(w), _p(s), _p(ray_id), M, n, _p(w_prefix), _p(w_total), _p(ws_prefix), _p(ws_total),
          _p(ws), ws.numel(), _s(w))
    return [w_prefix, w_total, ws_prefix, ws_total]


__all__ = ['cumdist_thres', 'segment_cumsum']
