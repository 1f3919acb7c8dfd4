"""CPU: the library's inline PTX lives in two headers -- k4_ptx.cuh (one definition of every sm_90 primitive but the
warpgroup MMAs) and k4_wgmma.cuh (the warpgroup MMAs) -- and build.py rebuilds the library when any header changes."""
import importlib.util
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, '4k-nerf_b200', 'csrc')
PTX_HEADERS = {'k4_ptx.cuh', 'k4_wgmma.cuh'}
ASM = re.compile(r'\b(?:asm|__asm__)\s*(?:volatile|__volatile__)?\s*\(')


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', '.h')))


def test_inline_ptx_only_in_the_primitive_headers():
    found = {}
    for f in sources():
        if f in PTX_HEADERS:
            continue
        for n, line in enumerate(open(os.path.join(CSRC, f)).read().splitlines(), 1):
            if ASM.search(line):
                found.setdefault(f, []).append(n)
    assert not found, f'inline PTX outside {sorted(PTX_HEADERS)} (file: lines): {found}'
    for f in PTX_HEADERS:
        assert ASM.search(open(os.path.join(CSRC, f)).read()), f


def test_build_tracks_every_header():
    spec = importlib.util.spec_from_file_location('k4_build', os.path.join(CSRC, 'build.py'))
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    headers = [f for f in sources() if f.endswith(('.cuh', '.h'))]
    assert 'k4_ptx.cuh' in headers
    missing = sorted(set(headers) - set(build.HEADERS))
    assert not missing, f'headers build.py does not rebuild on: {missing}'
