"""GPU: the distortion loss (csrc/k4_distloss.cu) -- torch_efficient_distloss.flatten_eff_distloss, its gradient,
ub360_utils_cuda.segment_cumsum and dcvgo.DistortionLoss -- against the float64 restatement
train_ref64.flatten_eff_distloss (autograd for the gradient) on sample-list layouts that stress the segmented scan.

Error model (u = 2^-24; every bound is fp64 arithmetic on the restatement's values; n_r = the sample's ray length):
  * each in-ray prefix or suffix of w or w*m is an fp32 summation tree over at most n_r terms (thread-sequential,
    warp and CTA scans, tile carries) plus the rounding of w*m: within (n_r + 4) u sum_j |term_j| of the fp64 one.
  * a loss term 2 w (m W<i - WM<i) + I/3 w^2 carries its prefixes' errors times 2|w| (|m|, 1), plus 5u of its
    magnitude mag_i = 2|w| (|m| sum_<i |w| + sum_<i |w m|) + I/3 w^2 (product, difference, FMA, I/3, the sum).
  * the reduction: in a tile every term passes through at most 8 (thread) + 5 (warp) + 7 (warps) = 20 fp32
    additions, tiles are summed in fp64: 24u sum_i mag_i; then / n and the rounding to fp32: 2u |L|.
  * the gradient g/n (2 m (W<i - W>i) + 2 (WM>i - WM<i) + 2/3 I w): the four sums' errors, 5u of the magnitude of the
    bracket, 2u for g/n and the product.
Each case prints its largest observed error as a fraction of its bound.
"""
import sys

import pytest
import torch

import train_ref64 as R

pytestmark = pytest.mark.gpu

U = R.U
F64 = torch.float64


# ---------------------------------------------------------------------------------------------------------------------
# layouts: (ray_id, w, m) on the device; m sorted within each ray, w >= 0 as the training forward's weights
# ---------------------------------------------------------------------------------------------------------------------
def _list(ids, lengths, dev, seed, w_scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    ids = torch.as_tensor(ids, dtype=torch.int64)
    lengths = torch.as_tensor(lengths, dtype=torch.int64)
    ray_id = torch.repeat_interleave(ids, lengths).to(dev)
    M = ray_id.numel()
    w = (torch.rand(M, generator=g) ** 2 * w_scale).to(dev)
    u = torch.rand(M, generator=g).to(dev)
    order = torch.argsort(ray_id.double() * 2 + u.double())            # m sorted within each ray
    m = u[order].contiguous()
    return ray_id.contiguous(), w.contiguous(), m


def layout(name, dev):
    """(ray_id, w, m, batch size): the batch size is the number of rays the training step shot (>= max id + 1)."""
    g = torch.Generator().manual_seed(7)
    if name == 'lengths':
        L = [257, 1, 1024, 32, 1_048_600, 33, 255, 1025, 31, 256, 1023, 1]
        return (*_list(range(len(L)), L, dev, 1), len(L))
    if name == 'one_sample_1M':
        n = 1_000_000
        return (*_list(range(n), [1] * n, dev, 2), n)
    if name == 'gaps':
        # no ray 0, interior gaps, and 2000 trailing rays of the batch without samples
        ids = torch.randperm(4999, generator=g)[:3000].sort().values + 1
        L = torch.randint(1, 61, (3000,), generator=g)
        return (*_list(ids, L, dev, 3), 7000)
    if name == 'M1':
        return (*_list([5], [1], dev, 4), 9)
    if name == 'odd':
        L = torch.randint(1, 60, (200,), generator=g)
        L[-1] += 5 * 2048 + 777 - int(L.sum())                              # M = 11017: no multiple of 32, 256, 2048
        assert int(L[-1]) > 2048                                            # and one ray across two tile boundaries
        return (*_list(range(200), L, dev, 5), 200)
    if name == 'over_2p24':
        L = torch.randint(1, 257, (140_000,), generator=g)
        L = L[:int((torch.cumsum(L, 0) < (1 << 24) + 50_000).sum()) + 1]
        assert int(L.sum()) > (1 << 24)
        return (*_list(range(L.numel()), L, dev, 6, w_scale=0.05), L.numel())
    raise ValueError(name)


LAYOUTS = ['lengths', 'one_sample_1M', 'gaps', 'M1', 'odd', 'over_2p24']


# ---------------------------------------------------------------------------------------------------------------------
# fp64 per-sample sums and the bounds
# ---------------------------------------------------------------------------------------------------------------------
class Sums:
    """In-ray exclusive prefixes and suffixes (fp64, padded [rays, longest] layout as train_ref64) and the bounds."""

    def __init__(self, ray_id, w, m, interval):
        n, pos, L = R._segment_positions(ray_id)
        self.n = n
        w, m = w.double(), m.double()
        wm = w * m
        counts = torch.bincount(ray_id, minlength=n)
        nr = counts[ray_id].double()

        def dense(v):
            return torch.zeros(n, L, dtype=F64, device=v.device).index_put((ray_id, pos), v)

        def pre(v):
            D = dense(v)
            return (torch.cumsum(D, 1) - D)[ray_id, pos]

        def suf(v):
            D = dense(v)
            return (D.flip(1).cumsum(1).flip(1) - D)[ray_id, pos]

        self.w, self.m, self.I = w, m, float(interval)
        self.Wp, self.WMp, self.Ws, self.WMs = pre(w), pre(wm), suf(w), suf(wm)
        Ap, AMp, As, AMs = pre(w.abs()), pre(wm.abs()), suf(w.abs()), suf(wm.abs())
        self.W_tot = torch.zeros(n, dtype=F64, device=w.device).index_add_(0, ray_id, w)
        self.WM_tot = torch.zeros(n, dtype=F64, device=w.device).index_add_(0, ray_id, wm)
        self.cnt = counts.double()
        self.A_tot = torch.zeros(n, dtype=F64, device=w.device).index_add_(0, ray_id, w.abs())
        self.AM_tot = torch.zeros(n, dtype=F64, device=w.device).index_add_(0, ray_id, wm.abs())
        c = (nr + 4) * U
        self.dWp, self.dWMp, self.dWs, self.dWMs = c * Ap, c * AMp, c * As, c * AMs
        I, aw, am = self.I, w.abs(), m.abs()
        mag = 2 * aw * (am * Ap + AMp) + I / 3 * w * w
        self.loss = (2 * w * (m * self.Wp - self.WMp)).sum() / n + I / 3 * (w * w).sum() / n
        e = 2 * aw * (am * self.dWp + self.dWMp) + 5 * U * mag
        self.loss_bound = float((e.sum() + 24 * U * mag.sum()) / n + 2 * U * self.loss.abs())
        self.bracket = 2 * m * (self.Wp - self.Ws) + 2 * (self.WMs - self.WMp) + (2 * I / 3) * w
        self.bracket_err = 2 * am * (self.dWp + self.dWs) + 2 * (self.dWMs + self.dWMp) + \
            5 * U * (2 * am * (Ap + As) + 2 * (AMs + AMp) + (2 * I / 3) * aw)

    def grad(self, g=1.0, divide=True):
        s = g / self.n if divide else g
        return s * self.bracket, abs(s) * (self.bracket_err + 2 * U * self.bracket.abs())


def _ratio(ours, ref, bound, name):
    err = (ours.double() - ref.double()).abs()
    b = torch.as_tensor(bound, dtype=F64, device=err.device).expand_as(err)
    assert torch.isfinite(ours).all(), name
    bad = err > b
    if bad.any():
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f'{name}: {int(bad.sum())} of {err.numel()} over their bound; first at {i}: ours '
                             f'{ours.reshape(-1)[i].item():.9g} ref {ref.reshape(-1)[i].item():.9g} bound {b.reshape(-1)[i].item():.3g}')
    pos = b > 0
    return float((err[pos] / b[pos]).max()) if pos.any() else 0.0


def _ours(w, m, interval, ray_id):
    from k4nerf.torch_efficient_distloss import flatten_eff_distloss
    wl = w.detach().clone().requires_grad_(True)
    loss = flatten_eff_distloss(wl, m, interval, ray_id)
    (gw,) = torch.autograd.grad(loss, wl)
    return loss.detach(), gw


# ---------------------------------------------------------------------------------------------------------------------
# layouts against the restatement
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', LAYOUTS)
def test_layout_matches_float64_restatement(cuda_device, name):
    from k4nerf import ub360_utils_cuda
    ray_id, w, m, _ = layout(name, cuda_device)
    interval = 1 / 128
    loss, gw = _ours(w, m, interval, ray_id)
    # the restatement: loss and autograd gradient in fp64
    w64 = w.double().requires_grad_(True)
    ref = R.flatten_eff_distloss(w64, m.double(), interval, ray_id)
    (g64,) = torch.autograd.grad(ref, w64)
    S = Sums(ray_id, w, m, interval)
    assert abs(float(S.loss) - float(ref)) <= 1e-12 * abs(float(ref)) + 1e-300
    worst = {'loss': _ratio(loss, ref.detach(), S.loss_bound, 'loss')}
    _, gb = S.grad()
    worst['grad'] = _ratio(gw, g64, gb, 'dL/dw')
    # segment_cumsum: exclusive prefixes and per-ray totals
    wp, wt, wsp, wst = ub360_utils_cuda.segment_cumsum(w, m, ray_id)
    assert wt.shape == (S.n,) and wst.shape == (S.n,)
    worst['w_prefix'] = _ratio(wp, S.Wp, S.dWp, 'w_prefix')
    worst['ws_prefix'] = _ratio(wsp, S.WMp, S.dWMp, 'ws_prefix')
    worst['w_total'] = _ratio(wt, S.W_tot, (S.cnt + 4) * U * S.A_tot, 'w_total')
    worst['ws_total'] = _ratio(wst, S.WM_tot, (S.cnt + 4) * U * S.AM_tot, 'ws_total')
    assert torch.equal(wt[S.cnt == 0], torch.zeros_like(wt[S.cnt == 0]))
    print(f'\n[distloss {name}] M={ray_id.numel()} n={S.n} worst observed/bound '
          + ' '.join(f'{k} {v:.3g}' for k, v in worst.items()))


def test_exact_operands_are_bit_identical_to_float64(cuda_device):
    """Dyadic w (multiples of 1/16, <= 1/8) and m (multiples of 1/8), interval 3/4 (interval/3 = 1/4), rays of up to 40
    samples across three tiles and 256 rays (a power of two divisor): every partial sum, product and the division is
    exact in fp32, so segment_cumsum, the loss and the gradient equal fp64 bit for bit."""
    from k4nerf import ub360_utils_cuda
    g = torch.Generator().manual_seed(11)
    L = torch.randint(0, 41, (256,), generator=g)
    L[-1] = 17
    ray_id = torch.repeat_interleave(torch.arange(256), L).to(cuda_device)
    M = ray_id.numel()
    assert M > 2 * 2048
    w = (torch.randint(0, 3, (M,), generator=g).float() / 16).to(cuda_device)
    u = torch.randint(0, 8, (M,), generator=g).double().to(cuda_device) / 8
    m = u[torch.argsort(ray_id.double() * 2 + u, stable=True)].float().contiguous()
    interval = 0.75
    S = Sums(ray_id, w, m, interval)
    loss, gw = _ours(w, m, interval, ray_id)
    assert loss.double() == S.loss
    assert torch.equal(gw.double(), S.grad()[0])
    wp, wt, wsp, wst = ub360_utils_cuda.segment_cumsum(w, m, ray_id)
    for ours, ref in ((wp, S.Wp), (wt, S.W_tot), (wsp, S.WMp), (wst, S.WM_tot)):
        assert torch.equal(ours.double(), ref)


def test_bounds_reject_wrong_definitions(cuda_device):
    """Each wrong definition, evaluated in fp64, lies outside twice the bound the layouts are held to: an
    inclusive prefix, the batch size as the divisor, no interval/3 term, a backward without the suffix terms."""
    from k4nerf import ub360_utils_cuda
    ray_id, w, m, batch = layout('gaps', cuda_device)
    interval = 1 / 128
    S = Sums(ray_id, w, m, interval)
    assert batch > S.n
    loss, gw = _ours(w, m, interval, ray_id)
    g_ref, gb = S.grad()
    wp = ub360_utils_cuda.segment_cumsum(w, m, ray_id)[0]
    wd = S.w
    wrong = {
        'inclusive prefix': (wp, S.Wp, S.Wp + wd, S.dWp),
        'divided by the batch size': (loss, S.loss, S.loss * S.n / batch, S.loss_bound),
        'no interval/3 term (loss)': (loss, S.loss, S.loss - interval / 3 * (wd * wd).sum() / S.n, S.loss_bound),
        'no interval/3 term (grad)': (gw, g_ref, g_ref - (2 / 3) * interval * wd / S.n, gb),
        'no suffix terms': (gw, g_ref, (2 * S.m * S.Wp - 2 * S.WMp + (2 / 3) * interval * wd) / S.n, gb),
    }
    for k, (ours, ref, bad, bound) in wrong.items():
        _ratio(ours, ref, bound, k)                                          # ours passes ...
        d = (bad.double() - ref.double()).abs()
        assert (d > 2 * torch.as_tensor(bound, dtype=F64, device=d.device)).any(), k     # ... the wrong one does not
        print(f'[distloss discrimination] {k}: max |wrong - ref| / bound '
              f'{float((d / torch.as_tensor(bound, dtype=F64, device=d.device).clamp_min(1e-300)).max()):.3g}')


def test_deterministic_and_no_host_sync(cuda_device):
    from k4nerf.torch_efficient_distloss import flatten_eff_distloss
    ray_id, w, m, _ = layout('odd', cuda_device)
    runs = [_ours(w, m, 1 / 128, ray_id) for _ in range(5)]
    for loss, gw in runs[1:]:
        assert torch.equal(loss, runs[0][0]) and torch.equal(gw, runs[0][1])
    iv_dev = torch.tensor([1 / 128], device=cuda_device)
    wl = w.clone().requires_grad_(True)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for iv in (1 / 128, iv_dev):
            loss = flatten_eff_distloss(wl, m, iv, ray_id)
            (gw,) = torch.autograd.grad(loss, wl)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert torch.equal(loss, runs[0][0]) and torch.equal(gw, runs[0][1])


def test_drop_in_modules(cuda_device, monkeypatch):
    import k4nerf
    from k4nerf import dcvgo
    monkeypatch.setitem(sys.modules, 'torch_efficient_distloss', k4nerf.torch_efficient_distloss)
    from torch_efficient_distloss import flatten_eff_distloss
    g = torch.Generator().manual_seed(3)
    ray_id = torch.repeat_interleave(torch.arange(256), torch.randint(1, 50, (256,), generator=g)).to(cuda_device)
    w = torch.rand(ray_id.numel(), generator=g).to(cuda_device)
    m = torch.rand(ray_id.numel(), generator=g).to(cuda_device)
    n_max = 48
    wa, wb = w.clone().requires_grad_(True), w.clone().requires_grad_(True)
    la = flatten_eff_distloss(wa, m, 1 / n_max, ray_id)
    lb = dcvgo.distortion_loss(wb, m, n_max, ray_id)
    la.backward()
    lb.backward()
    assert torch.equal(la, lb)
    assert torch.equal(wb.grad, wa.grad * 256)                  # lib/dcvgo.py:406: no 1/n (n = 256, exact)


def test_argument_errors_on_the_device(cuda_device):
    from k4nerf.torch_efficient_distloss import flatten_eff_distloss
    w = torch.rand(10, device=cuda_device)
    rid = torch.zeros(10, dtype=torch.int64, device=cuda_device)
    for args in ((w[::2], w[::2], 0.1, rid[::2]), (w, w.double(), 0.1, rid), (w, w, 0.1, rid.int()),
                 (w, w, torch.ones(2, device=cuda_device), rid), (w, w, 'x', rid), (w, w[:5], 0.1, rid),
                 (w[:0], w[:0], 0.1, rid[:0])):
        with pytest.raises(RuntimeError):
            flatten_eff_distloss(*args)


# ---------------------------------------------------------------------------------------------------------------------
# end to end: run_sr.py's composite loss with the distortion term from the new op on the library side
# ---------------------------------------------------------------------------------------------------------------------
E2E = ['mpi_relu_fog', 'mpi_gauss_fog', 'mpi_lkrelu_fog', 'mpi_relu_pe_randbkgd_shell', 'dcvgo_inside_fog',
       'dcvgo_outside_shell']


@pytest.fixture
def no_tf32():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize('cid', E2E)
def test_training_gradients_with_the_distortion_op(cuda_device, no_tf32, monkeypatch, cid):
    """test_gpu_train_grad.run_case with the library side's distortion term from k4nerf (the restatement, on CPU
    tensors, keeps train_ref64's): density, k0 and rgbnet gradients within train_ref64.Bounds."""
    from k4nerf.torch_efficient_distloss import flatten_eff_distloss
    import test_gpu_train_grad as TG
    orig, calls = R.flatten_eff_distloss, []

    def distloss(w, m, interval, ray_id):
        if w.is_cuda:
            calls.append(w.numel())
            return flatten_eff_distloss(w, m, interval, ray_id)
        return orig(w, m, interval, ray_id)
    monkeypatch.setattr(R, 'flatten_eff_distloss', distloss)
    worst, stats = TG.run_case(cid, cuda_device)
    assert len(calls) == 1 and calls[0] > 0
    print(f'\n[distloss e2e {cid}] worst observed/bound {max(worst.values()):.3g} ({max(worst, key=worst.get)}); {stats}')
