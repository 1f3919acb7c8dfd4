"""CPU: the row windows tests/test_gpu_sftnet_chain.py checks each decoder layer on, derived from the reference
module's structure."""
import k4nerf
from test_gpu_sftnet_chain import NUM_BLOCK, needed_rows, reference_ops


def test_needed_rows_follow_the_receptive_field():
    """15 dense blocks of five 3x3 convolutions each, conv_first and conv_body one row each, the x4 tail 1/2 + 3 x 1/4
    LR rows: conv_body's output bf is needed on 2 rows around the kept block and the model input on 79, which
    receptive_halo() rounds up to 80."""
    for scale in (4, 1):
        ops = reference_ops(NUM_BLOCK, scale)
        need = needed_rows(ops, 400, scale, 200, 201)
        assert need['bf'] == (198, 203) and need['sbody'] == (197, 204) and need['x'] == (121, 280)
        assert need['x4.4.2'] == (196, 205) and need['x1.4.2'] == (193, 208) and need['xc0.4.2'] == (192, 209)
        assert need['cond'] == need['feat'] == (122, 279)
        if scale == 4:
            assert need['up1'] == (398, 404) and need['up2'] == (798, 806) and need['hr'] == (799, 805)
        # clipped at the tile's edges
        edge = needed_rows(ops, 30, scale, 0, 2)
        assert edge['x'] == (0, 30) and edge['bf'] == (0, 4)
    assert k4nerf.SFTNet(3, 4).receptive_halo() == 80
