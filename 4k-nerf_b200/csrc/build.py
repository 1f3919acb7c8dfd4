"""Build libk4nerf.so (the C-ABI CUDA library, include/k4nerf.h) IN-TREE for sm_90a (H100).

    python 4k-nerf_b200/csrc/build.py [--force] [--verbose]

Plain nvcc on the .cu files, no torch headers (seconds, not minutes); the result is written to
4k-nerf_b200/k4nerf/libk4nerf.so, next to the package that loads it.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), 'k4nerf', 'libk4nerf.so')
SOURCES = ['k4_capi.cu', 'k4_march.cu', 'k4_march_ws.cu', 'k4_sr.cu', 'k4_ops.cu', 'k4_train.cu', 'k4_distloss.cu',
           'k4_metrics.cu', 'k4_video.cu', 'k4_train_march.cu', 'k4_lpips.cu', 'k4_png.cu',
           'k4_val.cu']
HEADERS = ['k4_internal.cuh', 'k4_march_common.cuh', 'k4_march_ray.cuh', 'k4_march_mma.cuh', 'k4_march_mlp.cuh',
           'k4_ptx.cuh', 'k4_wgmma.cuh', 'k4_ws_cfgs.h',
           '../../include/k4nerf.h']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC,-fvisibility=hidden', '--expt-relaxed-constexpr', '-Xptxas', '-v',
         '-ccbin', '/usr/bin/g++']


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(os.path.join(HERE, f)) > t for f in SOURCES + HEADERS + ['build.py'])


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objs = []
    logs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, src.replace('.cu', '.o'))
        cmd = [NVCC, *FLAGS, '-c', os.path.join(HERE, src), '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        logs.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f'nvcc failed on {src}')
    with open(os.path.join(HERE, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(logs))
    if verbose:
        print('\n'.join(logs))
    cmd = [NVCC, '-shared', '-o', OUT, *objs, '-ccbin', '/usr/bin/g++', '-Xlinker', '--exclude-libs,ALL']
    subprocess.check_call(cmd)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
