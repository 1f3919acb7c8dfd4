"""Generate the golden fixtures of the view-conditioned VC-Decoder, SFTNet(3, 4, 64, 5, 32, num_cond) with num_cond 63 and
64 (run where the reference checkout exists, like make_golden.py; the existing fixtures are not regenerated).

    python tests/golden/make_golden_cond.py

 sftnet_cond63_ref.pt / sftnet_cond64_ref.pt
                              the REFERENCE's own lib/sr_esrnet.py SFTNet(3, 4, 64, 5, 32, num_cond) (CPU, fp32) with
                              oracle.sftnet.random_state_dict(seed=3, num_cond=num_cond) loaded strict=True, on the
                              conditions of test_sftnet_cond.golden_inputs (the view embedding of seeded unit directions;
                              for 64 a depth-like map in front): one plain forward on 20x28 and one tile_process (tile 16,
                              pad 10) on 24x40 with a 3-D [num_cond, H, W] condition, the reference's contract.  Also the
                              reference module's state_dict key -> shape table.
 sftnet_cond64_pretrained_ref.pt
                              the 64-channel net with pretrained/RealESRNet_x4plus.pth loaded on top, strict=False, as
                              run_sr.py:663 does (CondNet is not in the checkpoint and keeps the seeded weights), on
                              test_sftnet_cond.pretrained_inputs.
"""
import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402,F401  (puts the repository, tests/ and the package on sys.path)
from oracle import sftnet  # noqa: E402
from test_sftnet_cond import golden_inputs, pretrained_inputs  # noqa: E402

REFERENCE = '/root/reference'


def _reference_net(num_cond):
    sys.path.insert(0, REFERENCE)
    from lib import sr_esrnet                       # the reference's own module
    torch.manual_seed(0)
    net = sr_esrnet.SFTNet(n_in_colors=3, scale=4, num_feat=64, num_block=5, num_grow_ch=32, num_cond=num_cond, dswise=False)
    net.load_state_dict(sftnet.random_state_dict(seed=3, num_cond=num_cond), strict=True)
    return net.eval()


def make_cond_golden(num_cond):
    net = _reference_net(num_cond)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    x, c, xt, ct = golden_inputs(num_cond)
    with torch.no_grad():
        y = net(x, c)
        with contextlib.redirect_stdout(io.StringIO()):
            yt = net.tile_process(xt, ct, tile_size=16, tile_pad=10)
    name = f'sftnet_cond{num_cond}_ref.pt'
    torch.save({'forward': y.clone(), 'tile_process': yt.clone(), 'state_dict_shapes': shapes, 'param_seed': 3,
                'num_cond': num_cond,
                'source': f'reference lib/sr_esrnet.py SFTNet(num_cond={num_cond}), torch {torch.__version__} CPU'},
               os.path.join(HERE, name))
    print(name, tuple(y.shape), tuple(yt.shape), len(shapes), 'keys')


def make_cond64_pretrained_golden():
    net = _reference_net(64)
    with contextlib.redirect_stdout(io.StringIO()):
        net.load_network(load_path=os.path.join(REFERENCE, 'pretrained', 'RealESRNet_x4plus.pth'), device='cpu',
                         strict=False)
    net.eval()
    x, c = pretrained_inputs()
    with torch.no_grad():
        y = net(x, c)
    torch.save({'forward': y.clone(), 'param_seed': 3, 'num_cond': 64,
                'source': 'reference lib/sr_esrnet.py SFTNet(num_cond=64) + pretrained/RealESRNet_x4plus.pth '
                          f'(strict=False), torch {torch.__version__} CPU'},
               os.path.join(HERE, 'sftnet_cond64_pretrained_ref.pt'))
    print('sftnet_cond64_pretrained_ref.pt', tuple(y.shape), float(y.min()), float(y.max()))


if __name__ == '__main__':
    make_cond_golden(63)
    make_cond_golden(64)
    make_cond64_pretrained_golden()
