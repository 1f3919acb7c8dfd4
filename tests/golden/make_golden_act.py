"""Generate the golden fixture of DirectMPIGO's gauss / lkrelu colour MLP (run where the reference checkout exists, like
make_golden_x1.py; the existing fixtures are not regenerated).

    python tests/golden/make_golden_act.py

 mpi_act_ref.pt   the reference's rgbnet Sequential of lib/dmpigo.py:96-105 -- Linear, act, Sequential(Linear, act),
                  Linear with ONE act instance -- built with the REFERENCE's own lib/act.py GaussianActivation(a=0.05)
                  and with nn.LeakyReLU(), on the CPU in fp32, for two shapes:
                    llff   15-64-64-3    (configs/llff: k0 9, no view / position frequencies; ws config 6)
                    cfg8   72-128-128-3  (k0 12, 4 view and 5 position frequencies; ws config 8)
                  Weights: nn.Linear's initialisation from torch.manual_seed, then for gauss W1/b1 and W2/b2 scaled so
                  that the pre-activations spread over a few a (mpi_act.scale_for_act).  Per case: the state_dict, the
                  inputs [128, dim0] and the outputs [128, 3].
 lib/dmpigo.py itself cannot be imported on a CPU-only machine (it JIT-builds the CUDA extension and needs
 torch_scatter), so only lib/act.py is loaded, from its file.
"""
import importlib.util
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from mpi_act import A_GAUSS, scale_for_act  # noqa: E402

REFERENCE = '/root/reference'
SHAPES = {'llff': dict(k0=9, vpe=0, spe=0, width=64), 'cfg8': dict(k0=12, vpe=4, spe=5, width=128)}
N = 128


def _reference_act_module():
    spec = importlib.util.spec_from_file_location('reference_lib_act', os.path.join(REFERENCE, 'lib', 'act.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def inputs(shape, seed):
    """k0 ~ N(0, 1), the position code of points in [-1, 1]^3, the view embedding of unit directions (lib/dmpigo.py:338-351)."""
    rng = np.random.default_rng(seed)

    def emb(v, nf):
        f = 2.0 ** np.arange(nf)
        return np.concatenate([v, np.sin(v[:, :, None] * f).reshape(N, -1), np.cos(v[:, :, None] * f).reshape(N, -1)], 1)
    d = rng.standard_normal((N, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x = np.concatenate([rng.standard_normal((N, shape['k0'])), emb(rng.uniform(-1, 1, (N, 3)), shape['spe']), emb(d, shape['vpe'])], 1)
    return torch.tensor(x, dtype=torch.float32)


def reference_rgbnet(act_mod, act_type, dim0, width, seed):
    act = act_mod.GaussianActivation(a=A_GAUSS) if act_type == 'gauss' else nn.LeakyReLU()
    torch.manual_seed(seed)
    net = nn.Sequential(nn.Linear(dim0, width), act, nn.Sequential(nn.Linear(width, width), act), nn.Linear(width, 3))
    nn.init.constant_(net[-1].bias, 0)
    return net


def main():
    act_mod = _reference_act_module()
    out = {'source': 'reference lib/act.py GaussianActivation / nn.LeakyReLU in the lib/dmpigo.py rgbnet Sequential, '
                     'torch %s CPU fp32' % torch.__version__, 'a': A_GAUSS, 'cases': {}}
    for si, (name, shape) in enumerate(SHAPES.items()):
        dim0 = shape['k0'] + 3 + 6 * shape['spe'] + 3 + 6 * shape['vpe']
        x = inputs(shape, seed=20 + si)
        for ai, act_type in enumerate(('gauss', 'lkrelu')):
            net = reference_rgbnet(act_mod, act_type, dim0, shape['width'], seed=30 + 10 * si + ai)
            lins = [net[0], net[2][0], net[3]]
            layers = [(l.weight.detach().double().numpy(), l.bias.detach().double().numpy()) for l in lins]
            with torch.no_grad():
                for l, (W, b) in zip(lins, scale_for_act(layers, x.double().numpy(), act_type)):
                    l.weight.copy_(torch.from_numpy(W))
                    l.bias.copy_(torch.from_numpy(b))
                y = net(x)
            sd = {k: v.clone() for k, v in net.state_dict().items()}
            out['cases'][f'{name}-{act_type}'] = {'shape': dict(shape, dim0=dim0), 'act_type': act_type, 'state_dict': sd,
                                                 'x': x.clone(), 'y': y.clone()}
            print(name, act_type, sorted(sd), tuple(y.shape), float(y.abs().max()))
    torch.save(out, os.path.join(HERE, 'mpi_act_ref.pt'))


if __name__ == '__main__':
    main()
