"""CPU: k4_testing_march_phases (the profiled ws marcher, include/k4nerf.h) reports bad arguments as K4_ERR_INVALID_ARG
before any CUDA call and leaves *n_ctas at 0; its slot constants match the header."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_enum(name):
    text = open(os.path.join(ROOT, 'include', 'k4nerf.h')).read()
    return int(re.search(rf'\b{name}\s*=\s*(\d+)', text).group(1))


def test_phase_slots_match_the_header():
    from k4nerf import _lib
    assert _lib.K4_PHASE_SLOTS == header_enum('K4_PHASE_SLOTS')
    for names, prefix in ((_lib.MARCHER_PHASES, 'K4_PH_M_'), (_lib.MLP_PHASES, 'K4_PH_L_')):
        for slot, nm in names.items():
            assert header_enum(prefix + nm.upper()) == slot, nm
    assert header_enum('K4_PH_ELAPSED') == 0
    assert header_enum('K4_PH_M_BATCHES') == header_enum('K4_PH_L_BATCHES') == _lib.K4_PHASE_SLOTS - 1


def test_march_phases_validates_arguments_without_a_gpu():
    """The scene is a zero-filled host block: a scene without an MLP, which is K4_ERR_UNSUPPORTED once the arguments are
    valid.  Nothing is dereferenced on the device before the checks."""
    from k4nerf import _lib
    lib = _lib.lib
    buf = C.create_string_buffer(256)
    p = C.addressof(buf)
    scene = C.create_string_buffer(1 << 16)
    out = _lib.RenderOut()
    out.d_rgb_marched = out.d_alphainv_last = p

    def call(sc=C.addressof(scene), mode=_lib.K4_MLP_TCGEN05_WS, n_rays=64, o=out, phases=p, max_ctas=132, args=True):
        a = _lib.RenderArgs()
        a.stepsize, a.mlp_mode = 0.5, mode
        n = C.c_int32(7)
        st = lib.k4_testing_march_phases(sc, C.byref(a) if args else None, p, p, p, n_rays, C.byref(o) if o else None,
                                         p, 256, phases, max_ctas, C.byref(n), None)
        return st, n.value

    for kw in (dict(sc=None), dict(args=False), dict(o=None), dict(phases=None), dict(max_ctas=0), dict(max_ctas=-1),
               dict(n_rays=0), dict(n_rays=-5), dict(mode=_lib.K4_MLP_TCGEN05), dict(mode=_lib.K4_MLP_FP32), dict(mode=5)):
        assert call(**kw) == (-1, 0), kw
    assert call() == (-2, 0)
