"""CPU: the fused training step accepts exactly the rgbnet shapes its kernels are sized for (k0 32, width 128, MLP input
128 = K4_MAX_DIM0) and rejects the next one up, in k4nerf.train_fused._model_shape and in the C ABI's checks, which
return before any CUDA call.  tests/test_gpu_train_fused_shapes.py runs the accepted limits on the GPU."""
import pytest

from test_train_fused import _both, _dvgo, _mpi, _valid

# (constructor, kwargs, MLP input width)
ACCEPTED = [
    (_mpi, dict(rgbnet_dim=32, spatial_pe=5, viewbase_pe=10, rgbnet_width=128), 128),
    (_dvgo, dict(rgbnet_dim=32, viewbase_pe=10, rgbnet_width=128, rgbnet_direct=True), 95),
    (_dvgo, dict(rgbnet_dim=32, viewbase_pe=10, rgbnet_width=128, rgbnet_direct=False), 92),
]
REJECTED = [
    (_mpi, dict(rgbnet_dim=27, spatial_pe=6, viewbase_pe=10, rgbnet_width=128), 129),
    (_mpi, dict(rgbnet_dim=32, spatial_pe=5, viewbase_pe=10, rgbnet_width=129), 128),
    (_dvgo, dict(rgbnet_dim=33, viewbase_pe=10, rgbnet_width=128, rgbnet_direct=True), 96),
    (_dvgo, dict(rgbnet_dim=12, viewbase_pe=11, rgbnet_width=128, rgbnet_direct=True), 81),
]


def _dim0(m):
    from k4nerf._scene import linear_layers
    return linear_layers(m.rgbnet)[0].in_features


@pytest.mark.parametrize('i', range(len(ACCEPTED)))
def test_model_shape_accepts_the_limits(i):
    from k4nerf.train_fused import _model_shape
    make, kw, dim0 = ACCEPTED[i]
    m = make(**kw)
    assert _dim0(m) == dim0
    kind, act, layers = _model_shape(m)
    assert len(layers) == 3 and layers[0].out_features == kw['rgbnet_width']


@pytest.mark.parametrize('i', range(len(REJECTED)))
def test_model_shape_rejects_past_the_limits(i):
    from k4nerf.train_fused import _model_shape
    make, kw, dim0 = REJECTED[i]
    m = make(**kw)
    assert _dim0(m) == dim0
    with pytest.raises(NotImplementedError):
        _model_shape(m)


def test_c_abi_rejects_mlp_input_129():
    """DirectMPIGO with k0 27, spatial_pe 6, viewbase_pe 10: input 27 + 39 + 63 = 129, one past K4_MAX_DIM0, with every
    other field within its limit."""
    import ctypes as C
    buf = C.create_string_buffer(1 << 12)
    ws = C.create_string_buffer(1 << 14)
    wsa = (C.addressof(ws) + 15) // 16 * 16
    a = _valid(buf, k0_dim=27, spatial_pe=6, viewbase_pe=10, rgbnet_width=128)
    assert _both(a, wsa, 8192) == (-2, -2)
