"""CPU: the C-ABI library loads and exports every symbol include/k4nerf.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, 'include', 'k4nerf.h')).read()
    return sorted(set(re.findall(r'K4_API\s+[A-Za-z_ \*]+?\b(k4_[a-z0-9_]+)\s*\(', text)))


def test_header_declares_expected_entry_points():
    syms = declared_symbols()
    for s in ('k4_scene_create', 'k4_scene_destroy', 'k4_render_rays', 'k4_render_workspace_bytes',
              'k4_make_rays', 'k4_abi_version', 'k4_status_string'):
        assert s in syms


def test_library_exports_every_declared_symbol():
    from k4nerf import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in declared_symbols():
        assert hasattr(lib, s), f'{s} declared in include/k4nerf.h but not exported'
    assert set(_lib.EXPORTS) <= set(declared_symbols())
    assert lib.k4_abi_version() == 1


def test_status_strings():
    from k4nerf import _lib
    assert _lib.lib.k4_status_string(0) == b'ok'
    assert b'unsupported' in _lib.lib.k4_status_string(-2)


def test_no_oracle_import_in_product():
    """The product package must never import the oracle (no CPU fallback)."""
    pkg = os.path.join(ROOT, '4k-nerf_b200')
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                src = open(os.path.join(dp, f)).read()
                assert 'import oracle' not in src and 'from oracle' not in src, f


def test_multi_gpu_entry_points_validate_arguments_without_a_gpu():
    """k4_render_rays_frames / k4_srnet_forward_roi_peers / k4_peer_*: argument errors are reported as status codes before
    any CUDA call (no compute here -- there is no GPU in the CPU test environment)."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    assert lib.k4_render_rays_frames(None, None, None, None, None, 0, None, None, None, 0, None) == -1       # K4_ERR_INVALID_ARG
    assert lib.k4_srnet_forward_roi_peers(None, None, None, 8, 8, 0, 8, 0, 8, None, 0, 0, 0, None, None, 0, None) == -1
    p = C.c_void_p()
    assert lib.k4_peer_alloc(0, C.byref(p)) == -1 and p.value is None
    assert lib.k4_peer_export(None, C.create_string_buffer(64)) == -1
    assert lib.k4_peer_open(None, C.byref(p)) == -1
    assert lib.k4_peer_free(None) == 0 and lib.k4_peer_close(None) == 0
    d = _lib.FrameDst()
    assert C.sizeof(d) == 4 * 4 + 8 + 8 * _lib.K4_MAX_PEERS                 # the header's k4_frame_dst, field for field


def test_testing_conv3x3_validates_arguments_without_a_gpu():
    """k4_testing_conv3x3 (one decoder convolution for the GPU tests): bad arguments are reported as K4_ERR_INVALID_ARG
    before any CUDA call, and *kernel_used says that nothing ran."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    A = _lib.ConvTestArgs
    assert C.sizeof(A) == 224 and A.out_plane_stride.offset == 160 and A.kernel.offset == 216     # the header's layout
    buf = C.create_string_buffer(64)                 # any non-null address: nothing is dereferenced before the checks

    def args(**kw):
        a = A()
        a.d_weight = a.d_bias = a.d_src = a.d_dst_h = C.addressof(buf)
        a.cout, a.cin, a.src_cstride, a.H, a.W, a.y_lo, a.y_hi, a.dst_cstride = 64, 64, 64, 8, 8, 0, 8, 64
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    used = C.c_int32(7)
    bad = [dict(d_weight=None), dict(d_bias=None), dict(d_src=None), dict(d_dst_h=None), dict(y_lo=5, y_hi=4),
           dict(y_lo=3, y_hi=3), dict(y_hi=9), dict(y_lo=-1), dict(mode=8), dict(mode=-1), dict(kernel=4), dict(kernel=-1),
           dict(cout=0), dict(cout=65), dict(cin=193), dict(H=0), dict(src_cstride=60), dict(src_c0=4, src_cstride=72),
           dict(src_cstride=32), dict(dst_c0=8), dict(mode=1), dict(mode=3), dict(mode=4),
           dict(mode=5), dict(mode=7, d_dst_f=C.addressof(buf))]
    for kw in bad:
        used.value = 7
        assert lib.k4_testing_conv3x3(C.byref(args(**kw)), C.byref(used), None) == -1, kw
        assert used.value == -1, kw
    assert lib.k4_testing_conv3x3(None, C.byref(used), None) == -1
    # combinations the decoder does not build: the fused SFT epilogues after a 16-channel or an upsampling layer
    ptrs = (C.c_void_p * 8)(*([C.addressof(buf)] * 8))
    sft = dict(mode=5, d_cond16=C.addressof(buf), h_sft=C.cast(ptrs, C.POINTER(C.c_void_p)))
    assert lib.k4_testing_conv3x3(C.byref(args(cout=16, **sft)), C.byref(used), None) == -2
    assert lib.k4_testing_conv3x3(C.byref(args(upsample2x=1, **sft)), C.byref(used), None) == -2
