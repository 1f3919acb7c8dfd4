"""numpy restatements of csrc/k4_val.cu's MSE for the tests: numpy's pairwise float32 sum evaluated the way the kernel
evaluates it (the units at the depth of the first leaf, each unit's subtree, then the perfect tree above them), and
the element order of ``a - b`` that k4nerf.utils.numpy_visit_order gives the kernel."""
import numpy as np

from k4nerf.utils import numpy_visit_order

f32 = np.float32


def split(s):
    h = s // 2
    return h - h % 8


def plan(n):
    """(U, depth of the deepest unit subtree) of numpy's pairwise tree over n values."""
    sizes, depth, U, below = {n}, 0, None, None
    while sizes:
        if U is None and any(s <= 128 for s in sizes):
            U, below = depth, 0
        elif U is not None:
            below += 1
        sizes = {c for s in sizes if s > 128 for c in (split(s), s - split(s))}
        depth += 1
    return U, below


def _leaf_sums(x, lo, s):
    """pairwise_sum's leaf (s <= 128 values from lo) for arrays of leaves of one size s."""
    blk = x[lo[:, None] + np.arange(s)[None, :]]
    if s < 8:
        r = np.full(lo.size, -0.0, f32)
        for i in range(s):
            r = (r + blk[:, i]).astype(f32)
        return r
    r = blk[:, :8].copy()
    for i in range(8, s - s % 8, 8):
        r = (r + blk[:, i:i + 8]).astype(f32)
    res = (((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))).astype(f32)
    for i in range(s - s % 8, s):
        res = (res + blk[:, i]).astype(f32)
    return res


def _node_sums(x, lo, s):
    """Sums of the subtrees at (lo[i], s[i]): leaves directly, larger nodes through their two children."""
    out = np.empty(lo.size, f32)
    leaf = s <= 128
    for m in np.unique(s[leaf]):
        sel = np.nonzero(leaf & (s == m))[0]
        out[sel] = _leaf_sums(x, lo[sel], int(m))
    inner = np.nonzero(~leaf)[0]
    if inner.size:
        h = s[inner] // 2
        h -= h % 8
        left = _node_sums(x, lo[inner], h)
        right = _node_sums(x, lo[inner] + h, s[inner] - h)
        out[inner] = (left + right).astype(f32)
    return out


def pairwise_sum(x):
    """numpy's pairwise_sum of a 1-D float32 array, evaluated unit by unit and then as a perfect tree."""
    x = np.ascontiguousarray(x, dtype=f32)
    U, _ = plan(x.size)
    lo, s = np.zeros(1, np.int64), np.array([x.size], np.int64)
    for _ in range(U):
        h = s // 2
        h -= h % 8
        lo = np.stack([lo, lo + h], 1).ravel()
        s = np.stack([h, s - h], 1).ravel()
    v = _node_sums(x, lo, s)
    while v.size > 1:
        v = (v[0::2] + v[1::2]).astype(f32)
    return v[0]


def mse_np(a, b):
    """np.mean(np.square(a - b)) of float32 [H, W, 3] arrays as the kernel computes it, from the operands' strides."""
    order = numpy_visit_order(a.shape, [s // a.itemsize for s in a.strides], [s // b.itemsize for s in b.strides])
    d = np.square((np.transpose(a, order) - np.transpose(b, order)).astype(f32)).astype(f32).ravel()
    total = f32(f32(0.0) + pairwise_sum(d))
    return f32(np.float64(total) / np.float64(d.size))
