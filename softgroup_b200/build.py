"""Compile softgroup_b200/csrc/*.cu into softgroup_b200/libsgb200.so (sm_90a only, in-tree).

nvcc cross-compiles without a GPU. The .so and the objects under csrc/build/ are build products (git-ignored).
"""
import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, 'csrc', 'build')
LIB = os.path.join(HERE, 'libsgb200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
    '--expt-relaxed-constexpr'
]


def _newer(src, dst):
    return (not os.path.exists(dst)) or os.path.getmtime(src) > os.path.getmtime(dst)


def build(force=False, verbose=False):
    srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')))
    hdrs = glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(HERE, '..', 'include', '*.h'))
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = max(os.path.getmtime(h) for h in hdrs)
    jobs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + '.o')
        if force or _newer(s, o) or os.path.getmtime(o) < hdr_time:
            jobs.append((s, o))

    def run(job):
        s, o = job
        cmd = [NVCC] + FLAGS + ['-c', s, '-o', o]
        if verbose:
            print(' '.join(cmd), file=sys.stderr)
        subprocess.check_call(cmd)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, os.path.basename(s)[:-3] + '.o') for s in srcs]
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-cudart', 'static']
        if verbose:
            print(' '.join(cmd), file=sys.stderr)
        subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='-f' in sys.argv, verbose=True))
