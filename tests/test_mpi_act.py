"""CPU: DirectMPIGO's act_type 'gauss' / 'lkrelu' (lib/dmpigo.py:89-95) on the host side -- the module against the
reference's own Sequential (tests/golden/mpi_act_ref.pt, from lib/act.py), state_dict keys, checkpoint round trip, the
ctypes mirror of k4_scene_desc and the arguments k4_scene_create refuses."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import mpi_act

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = torch.load(os.path.join(HERE, 'golden', 'mpi_act_ref.pt'), weights_only=False)
CASES = sorted(GOLDEN['cases'])


def _model(act_type, k0=9, vpe=0, spe=0, width=64):
    import k4nerf
    return k4nerf.DirectMPIGO(xyz_min=[-1, -1, -1], xyz_max=[1, 1, 1], num_voxels=8 * 8 * 8, mpi_depth=8,
                              rgbnet_dim=k0, rgbnet_depth=3, rgbnet_width=width, viewbase_pe=vpe, spatial_pe=spe,
                              act_type=act_type, mode_type='mlp')


def _layers(sd):
    return [(sd[k + '.weight'], sd[k + '.bias']) for k in ('0', '2.0', '3')]


@pytest.mark.parametrize('case', CASES)
def test_golden_exercises_the_activation(case):
    c = GOLDEN['cases'][case]
    layers = [(W.double().numpy(), b.double().numpy()) for W, b in _layers(c['state_dict'])]
    mpi_act.assert_exercised(layers, c['x'].double().numpy(), c['act_type'])


@pytest.mark.parametrize('case', CASES)
def test_oracle_mlp_matches_reference_sequential(case):
    c = GOLDEN['cases'][case]
    y = mpi_act.mlp_act(_layers(c['state_dict']), c['x'], c['act_type'], GOLDEN['a'])
    assert torch.allclose(y, c['y'], rtol=1e-5, atol=1e-6), float((y - c['y']).abs().max())
    # and the fp64 evaluation of the same expression is within float tolerance
    y64 = mpi_act.mlp_act([(W.double(), b.double()) for W, b in _layers(c['state_dict'])], c['x'].double(), c['act_type'])
    assert torch.allclose(y64, c['y'].double(), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize('case', CASES)
def test_module_rgbnet_matches_reference(case):
    c = GOLDEN['cases'][case]
    s = c['shape']
    m = _model(c['act_type'], s['k0'], s['vpe'], s['spe'], s['width'])
    assert m.dim0 == s['dim0']
    m.rgbnet.load_state_dict(c['state_dict'])
    with torch.no_grad():
        y = m.rgbnet(c['x'])
    assert torch.allclose(y, c['y'], rtol=1e-5, atol=1e-6), float((y - c['y']).abs().max())


@pytest.mark.parametrize('case', CASES)
def test_state_dict_keys_and_shapes_equal_reference(case):
    c = GOLDEN['cases'][case]
    s = c['shape']
    m = _model(c['act_type'], s['k0'], s['vpe'], s['spe'], s['width'])
    ours = {k: tuple(v.shape) for k, v in m.rgbnet.state_dict().items()}
    ref = {k: tuple(v.shape) for k, v in c['state_dict'].items()}
    assert ours == ref
    if c['act_type'] == 'gauss':
        # one shared GaussianActivation after every hidden Linear: both keys, one parameter, frozen
        assert {'1.a', '2.1.a'} <= set(ours)
        assert m.rgbnet[1] is m.rgbnet[2][1]
        assert not m.rgbnet[1].a.requires_grad and float(m.rgbnet[1].a) == pytest.approx(0.05)


@pytest.mark.parametrize('act_type', ['relu', 'gauss', 'lkrelu'])
def test_checkpoint_round_trip_through_load_model(tmp_path, act_type):
    from k4nerf import dmpigo, utils
    m = _model(act_type)
    with torch.no_grad():
        for p in m.rgbnet.parameters():
            p.add_(torch.randn_like(p) * 0.01)
        if act_type == 'gauss':
            m.rgbnet[1].a.fill_(0.07)
    path = tmp_path / 'fine_last.tar'
    torch.save({'global_step': 1, 'model_kwargs': m.get_kwargs(), 'model_state_dict': m.state_dict()}, path)
    m2 = utils.load_model(dmpigo.DirectMPIGO, str(path))
    assert m2.act_type == act_type
    sd1, sd2 = m.state_dict(), m2.state_dict()
    assert sd1.keys() == sd2.keys() and all(torch.equal(sd1[k], sd2[k]) for k in sd1)
    extra = m2._scene_extra()
    assert extra['rgbnet_act'] == mpi_act.K4_ACT[act_type]
    if act_type == 'gauss':
        assert float(extra['rgbnet_act_param']) == pytest.approx(0.07)
    else:
        assert extra['rgbnet_act_param'] is None


def test_unknown_act_type_is_a_value_error():
    with pytest.raises(ValueError, match="'relu', 'gauss', 'lkrelu'"):
        _model('elu')


def test_scene_desc_mirror_offsets_match_the_header(tmp_path):
    """The ctypes SceneDesc against the C compiler's layout of include/k4nerf.h's k4_scene_desc."""
    from k4nerf import _lib
    fields = [f[0] for f in _lib.SceneDesc._fields_]
    assert fields[fields.index('spatial_pe') + 1] == 'rgbnet_act' and fields[-1] == 'rgbnet_act_param'
    src = tmp_path / 'off.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "k4nerf.h"\nint main(void) {\n'
                   + ''.join(f'  printf("{f} %zu\\n", offsetof(k4_scene_desc, {f}));\n' for f in fields)
                   + '  printf("sizeof %zu\\n", sizeof(k4_scene_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'off'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for f in fields:
        assert int(got[f]) == getattr(_lib.SceneDesc, f).offset, f
    assert int(got['sizeof']) == C.sizeof(_lib.SceneDesc)
    assert (_lib.K4_ACT_RELU, _lib.K4_ACT_GAUSS, _lib.K4_ACT_LKRELU) == (0, 1, 2)


@pytest.mark.parametrize('kind,act,a', [(1, 3, 0.05), (1, -1, 0.05), (0, 1, 0.05), (2, 2, 0.0), (1, 1, 0.0),
                                        (1, 1, -0.05), (1, 1, float('nan')), (1, 1, float('inf'))])
def test_scene_create_refuses_bad_activations(kind, act, a):
    """An unknown activation, a gauss / lkrelu one on DirectVoxGO or DirectContractedVoxGO, a Gaussian's a that is not
    finite and > 0: K4_ERR_INVALID_ARG, checked before any device work (so also on a machine without a GPU)."""
    from k4nerf import _lib
    d = _lib.SceneDesc()
    d.kind = kind
    d.world_size[:] = [8, 8, 8]
    d.mask_size[:] = [8, 8, 8]
    d.k0_dim = 9
    d.mpi_depth = 8
    d.d_density = d.d_k0 = d.d_mask = d.d_act_shift_grid = 16       # never dereferenced: refused first
    d.rgbnet_act = act
    d.rgbnet_act_param = a
    out = C.c_void_p()
    assert _lib.lib.k4_scene_create(C.byref(d), None, C.byref(out)) == -1
    assert not out.value


def test_bound_helpers_reduce_to_relu():
    """The fp64 error model with act='relu' is march_bounds' model (the activation step adds nothing)."""
    from types import SimpleNamespace
    import march_bounds
    rng = np.random.default_rng(0)
    spec = ('x', 'cfgB', 9, 0, 0, 64, 1, 6)
    m = march_bounds.shape_info(SimpleNamespace(), spec)
    m.layers = [(rng.standard_normal((64, 15)) * 0.3, rng.standard_normal(64) * 0.1),
                (rng.standard_normal((64, 64)) * 0.1, rng.standard_normal(64) * 0.1),
                (rng.standard_normal((3, 64)) * 0.1, np.zeros(3))]
    x = rng.standard_normal((50, 15))
    for mode in ('fp32', 'f16x3'):
        a = march_bounds.logit_bound(mode, m, x, None)
        b = mpi_act.act_logit_bound(mode, m, x, None, 'relu')
        assert np.allclose(a[0], b[0]) and np.allclose(a[1], b[1], rtol=1e-12)
    for mode in ('f16', 'ws', 'fp32'):
        a = march_bounds.true_logit_bound(mode, m, x, None)
        b = mpi_act.act_logit_bound(mode, m, x, None, 'relu', true=True)
        assert np.allclose(a[0], b[0]) and np.allclose(a[1], b[1], rtol=1e-12)
