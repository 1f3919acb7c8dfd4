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
              'k4_make_rays', 'k4_abi_version', 'k4_status_string', 'k4_png_encode', 'k4_testing_png_code_lengths'):
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


def test_testing_condnet_validates_arguments_without_a_gpu():
    """k4_testing_condnet (CondNet on a row window for the GPU tests): bad arguments are reported as K4_ERR_INVALID_ARG
    before any CUDA call, and *kernel_used says that nothing ran."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    A = _lib.CondnetTestArgs
    assert C.sizeof(A) == 56 and A.H.offset == 16 and A.d_cond_out.offset == 32 and A.kernel.offset == 48   # the header's layout
    buf = C.create_string_buffer(64)
    ptrs = (C.c_void_p * 8)(*([C.addressof(buf)] * 8))
    holey = (C.c_void_p * 8)(*([C.addressof(buf)] * 7 + [None]))

    def args(**kw):
        a = A()
        a.h_condnet = C.cast(ptrs, C.POINTER(C.c_void_p))
        a.d_cond_in = a.d_cond_out = a.d_cond16 = C.addressof(buf)
        a.H, a.W, a.y_lo, a.y_hi = 8, 8, 0, 8
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    used = C.c_int32(7)
    bad = [dict(h_condnet=None), dict(h_condnet=C.cast(holey, C.POINTER(C.c_void_p))), dict(d_cond_in=None),
           dict(d_cond_out=None), dict(H=0), dict(W=0), dict(H=1 << 16, W=1 << 15), dict(y_lo=5, y_hi=4),
           dict(y_lo=3, y_hi=3), dict(y_hi=9), dict(y_lo=-1), dict(kernel=3), dict(kernel=-1),
           dict(d_cond_out=C.addressof(buf) + 4), dict(d_cond16=C.addressof(buf) + 2), dict(d_cond_in=C.addressof(buf) + 1)]
    for kw in bad:
        used.value = 7
        assert lib.k4_testing_condnet(C.byref(args(**kw)), C.byref(used), None) == -1, kw
        assert used.value == -1, kw
    assert lib.k4_testing_condnet(None, C.byref(used), None) == -1


def test_testing_sft_validates_arguments_without_a_gpu():
    """k4_testing_sft (one SFT layer as its own pass for the GPU tests): bad arguments are reported as K4_ERR_INVALID_ARG
    before any CUDA call, and *kernel_used says that nothing ran."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    A = _lib.SftTestArgs
    assert C.sizeof(A) == 104 and A.d_cond.offset == 16 and A.xh_cstride.offset == 40 and A.d_dst_f.offset == 64
    assert A.res_scale.offset == 80 and A.p0.offset == 88 and A.P.offset == 96                          # the header's layout
    buf = C.create_string_buffer(64)
    ptrs = (C.c_void_p * 8)(*([C.addressof(buf)] * 8))
    holey = (C.c_void_p * 8)(*([None] + [C.addressof(buf)] * 7))

    def args(**kw):
        a = A()
        a.h_sft = C.cast(ptrs, C.POINTER(C.c_void_p))
        a.d_cond = a.d_x_h = a.d_dst_h = C.addressof(buf)
        a.cout, a.xh_cstride, a.xh_c0, a.dst_cstride, a.dst_c0, a.p0, a.P = 32, 192, 160, 192, 160, 58, 406
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    used = C.c_int32(7)
    b = C.addressof(buf)
    bad = [dict(h_sft=None), dict(h_sft=C.cast(holey, C.POINTER(C.c_void_p))), dict(d_cond=None), dict(cout=16),
           dict(cout=48), dict(kernel=3), dict(kernel=-1), dict(p0=-1), dict(P=0), dict(P=(1 << 30) + 1),
           dict(d_x_h=None), dict(d_x_f=b), dict(d_dst_h=None), dict(d_dst_f=b, d_res_f=b),
           dict(d_dst_h=None, d_dst_f=b), dict(xh_c0=161), dict(xh_cstride=191), dict(xh_c0=-2), dict(cout=64),
           dict(dst_c0=164), dict(dst_cstride=196), dict(d_cond=b + 8), dict(d_x_h=b + 2), dict(d_dst_h=b + 8),
           dict(d_dst_h=None, d_dst_f=b + 4, d_res_f=b), dict(d_dst_h=None, d_dst_f=b, d_res_f=b + 4)]
    for kw in bad:
        used.value = 7
        assert lib.k4_testing_sft(C.byref(args(**kw)), C.byref(used), None) == -1, kw
        assert used.value == -1, kw
    assert lib.k4_testing_sft(None, C.byref(used), None) == -1


def test_testing_rgbnet_validates_arguments_without_a_gpu():
    """k4_testing_rgbnet (a scene's rgbnet on caller rows for the GPU tests): bad arguments are reported as
    K4_ERR_INVALID_ARG before any CUDA call, and *group_rows stays 0.  The scene here is a zero-filled host block: a scene
    without an MLP, whose every mode is K4_ERR_UNSUPPORTED once the arguments are valid."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    A = _lib.RgbnetTestArgs
    assert C.sizeof(A) == 56 and A.n.offset == 8 and A.d_x.offset == 16 and A.d_racc.offset == 48     # the header's layout
    buf = C.create_string_buffer(64)
    scene = C.create_string_buffer(1 << 16)           # zeros: kind DVGO, rgbnet_direct 0 -> d_diffuse required

    def args(**kw):
        a = A()
        a.mode, a.n = _lib.K4_MLP_F16, 33
        a.d_x = a.d_diffuse = a.d_w = a.d_owner = a.d_racc = C.addressof(buf)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    g = C.c_int32(7)
    bad = [dict(mode=-1), dict(mode=5), dict(n=0), dict(n=-3), dict(n=(1 << 24) + 1), dict(d_x=None), dict(d_w=None),
           dict(d_owner=None), dict(d_racc=None), dict(d_diffuse=None)]
    for kw in bad:
        g.value = 7
        assert lib.k4_testing_rgbnet(C.addressof(scene), C.byref(args(**kw)), C.byref(g), None) == -1, kw
        assert g.value == 0, kw
    assert lib.k4_testing_rgbnet(None, C.byref(args()), C.byref(g), None) == -1
    assert lib.k4_testing_rgbnet(C.addressof(scene), None, C.byref(g), None) == -1
    for mode in range(5):
        assert lib.k4_testing_rgbnet(C.addressof(scene), C.byref(args(mode=mode)), C.byref(g), None) == -2, mode
        assert g.value == 0


def test_testing_skip_field_validates_arguments_without_a_gpu():
    """k4_testing_skip_field (the empty-space-skipping field for the GPU tests): bad arguments are reported as
    K4_ERR_INVALID_ARG before any CUDA call, and cdims is zeroed.  The scene here is a zero-filled host block: a scene
    without a field, which is K4_ERR_UNSUPPORTED once the arguments are valid."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    buf = C.create_string_buffer(64)
    scene = C.create_string_buffer(1 << 16)
    cd = (C.c_int32 * 3)(7, 7, 7)
    for sc, out, n, dims in ((None, buf, 64, cd), (scene, None, 64, cd), (scene, buf, 0, cd), (scene, buf, -5, cd),
                             (scene, buf, 64, None)):
        cd[:] = [7, 7, 7]
        assert lib.k4_testing_skip_field(sc and C.addressof(sc), out and C.addressof(out), n, dims) == -1, (sc, out, n, dims)
        if dims is not None:
            assert list(cd) == [0, 0, 0]
    cd[:] = [7, 7, 7]
    assert lib.k4_testing_skip_field(C.addressof(scene), C.addressof(buf), 64, cd) == -2
    assert list(cd) == [0, 0, 0]


def test_testing_png_code_lengths_validates_arguments_without_a_gpu():
    """k4_testing_png_code_lengths (the PNG encoder's code lengths of a histogram, for the GPU tests): a NULL buffer,
    n outside 1..286 or maxbits outside 1..15 is K4_ERR_INVALID_ARG before any CUDA call."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    f = C.addressof(C.create_string_buffer(4 * 300))
    ln = C.addressof(C.create_string_buffer(300))
    for args in ((None, 19, 7, ln), (f, 19, 7, None), (f, 0, 7, ln), (f, -1, 7, ln), (f, 287, 15, ln), (f, 30, 0, ln),
                 (f, 30, 16, ln), (f, 30, -3, ln)):
        assert lib.k4_testing_png_code_lengths(*args, None) == -1, args


def test_testing_srnet_forward_upto_validates_arguments_without_a_gpu():
    """k4_testing_srnet_forward_upto (the decoder forward stopped after k steps, for the GPU tests): bad arguments are
    reported as K4_ERR_INVALID_ARG before any CUDA call, with *n_steps 0.  The net here is a zero-filled host block; every
    case has an invalid argument, so nothing reads it."""
    from k4nerf import _lib
    C = ctypes
    lib = _lib.lib
    assert C.sizeof(_lib.SrStep) == 20 and _lib.SrStep.fused.offset == 16                     # the header's layout
    assert C.sizeof(_lib.SrWsLayout) == 14 * 8 and _lib.SrWsLayout.cond16.offset == 16 and _lib.SrWsLayout.hr.offset == 96
    assert _lib.SR_STEP_KINDS.index('last') == 12 and _lib.SR_STEP_KINDS.index('sft_rrdb') == 6
    buf = C.create_string_buffer(64)
    net = C.create_string_buffer(1 << 16)
    steps = (_lib.SrStep * 4)()
    ns = C.c_int32(7)
    lay = _lib.SrWsLayout()

    def call(**kw):
        a = dict(net=C.addressof(net), x=C.addressof(buf), cond=C.addressof(buf), h=8, w=8, keep=(0, 8, 0, 8),
                 out=C.addressof(buf), ws=C.addressof(buf), ws_bytes=64, stop_after=1, steps=steps, max_steps=4,
                 n_steps=C.byref(ns), layout=C.byref(lay))
        a.update(kw)
        ns.value = 7
        return lib.k4_testing_srnet_forward_upto(a['net'], a['x'], a['cond'], a['h'], a['w'], *a['keep'], a['out'], 64, 8,
                                                 a['ws'], a['ws_bytes'], a['stop_after'], a['steps'], a['max_steps'],
                                                 a['n_steps'], a['layout'], None)

    bad = [dict(net=None), dict(stop_after=0), dict(stop_after=-1), dict(max_steps=-1), dict(steps=None),
           dict(layout=None), dict(h=0), dict(w=-2), dict(net=None, x=None)]
    for kw in bad:
        assert call(**kw) == -1, kw
        assert ns.value == 0, kw
    assert call(n_steps=None) == -1
