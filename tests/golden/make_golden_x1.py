"""Generate the golden fixtures of the x1 VC-Decoder (run where the reference checkout exists, like make_golden.py,
whose input generators it reuses; the existing fixtures are not regenerated).

    python tests/golden/make_golden_x1.py

 sftnet_x1_ref.pt             the REFERENCE's own lib/sr_esrnet.py SFTNet(3, 1, 64, 5, 32, 1) (CPU, fp32) with
                              test_sftnet_x1.x1_state_dict(seed=3) (the seeded
                              x4 set without conv_up1 / conv_up2) loaded strict=True, on the inputs of
                              sftnet_ref.pt: one plain forward on 20x28 and one tile_process (tile 16, pad 10) on 24x40.
                              Also the reference module's state_dict key -> shape table, so that key parity can be
                              checked without the reference checkout.
 sftnet_x1_pretrained_ref.pt  the same net with pretrained/RealESRNet_x4plus.pth loaded on top, strict=False, as
                              run_sr.py:663 does (conv_up1 / conv_up2 of the checkpoint are unexpected keys and dropped),
                              on the inputs of sftnet_pretrained_ref.pt.
"""
import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import sftnet_inputs, sftnet_pretrained_inputs  # noqa: E402  (also puts the repository on sys.path)
from test_sftnet_x1 import x1_state_dict  # noqa: E402

REFERENCE = '/root/reference'


def _reference_x1_net():
    sys.path.insert(0, REFERENCE)
    from lib import sr_esrnet                       # the reference's own module
    torch.manual_seed(0)
    net = sr_esrnet.SFTNet(n_in_colors=3, scale=1, num_feat=64, num_block=5, num_grow_ch=32, num_cond=1, dswise=False)
    net.load_state_dict(x1_state_dict(seed=3), strict=True)
    return net.eval()


def make_sftnet_x1_golden():
    net = _reference_x1_net()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    x, c, xt, ct = sftnet_inputs()
    with torch.no_grad():
        y = net(x, c)
        with contextlib.redirect_stdout(io.StringIO()):
            yt = net.tile_process(xt, ct, tile_size=16, tile_pad=10)
    torch.save({'forward': y.clone(), 'tile_process': yt.clone(), 'state_dict_shapes': shapes, 'param_seed': 3,
                'input_seed': 11, 'source': 'reference lib/sr_esrnet.py SFTNet(scale=1), torch %s CPU' % torch.__version__},
               os.path.join(HERE, 'sftnet_x1_ref.pt'))
    print('sftnet_x1_ref.pt', tuple(y.shape), tuple(yt.shape), len(shapes), 'keys')


def make_sftnet_x1_pretrained_golden():
    net = _reference_x1_net()
    with contextlib.redirect_stdout(io.StringIO()):
        net.load_network(load_path=os.path.join(REFERENCE, 'pretrained', 'RealESRNet_x4plus.pth'), device='cpu',
                         strict=False)
    net.eval()
    x, c = sftnet_pretrained_inputs()
    with torch.no_grad():
        y = net(x, c)
    torch.save({'forward': y.clone(), 'param_seed': 3, 'input_seed': 12,
                'source': 'reference lib/sr_esrnet.py SFTNet(scale=1) + pretrained/RealESRNet_x4plus.pth (strict=False), '
                          'torch %s CPU' % torch.__version__},
               os.path.join(HERE, 'sftnet_x1_pretrained_ref.pt'))
    print('sftnet_x1_pretrained_ref.pt', tuple(y.shape), float(y.min()), float(y.max()))


if __name__ == '__main__':
    make_sftnet_x1_golden()
    make_sftnet_x1_pretrained_golden()
