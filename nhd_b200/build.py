"""Builds nhd_b200/libnhd_b200.so (the C-ABI library with the sm_90a kernels) in-tree.

nvcc cross-compiles without a GPU; the resulting .so is a build product (git-ignored) that
_lib.py loads from the package directory."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libnhd_b200.so')
SOURCES = [os.path.join(CSRC, 'nhd_api.cu'), os.path.join(CSRC, 'nhd_ingest.cpp')]
DEPS = SOURCES + [os.path.join(CSRC, f) for f in ('nhd_kernels.cuh', 'nhd_core.cuh')] + \
    [os.path.join(HERE, '..', 'include', 'nhd_b200.h'), os.path.abspath(__file__)]   # this file: the nvcc flags
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '--fmad=false']                   # fp64 NIC arithmetic must stay subtract-then-compare (no contraction)


def nvcc_path():
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found')


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, profile=False, checks=False):
    if checks:
        return _compile(os.path.join(HERE, 'libnhd_b200_chk.so'), verbose, ['-DNHD_CHECKS'])
    if profile:
        return _compile(os.path.join(HERE, 'libnhd_b200_prof.so'), verbose, ['-DNHD_PROFILE'])
    if not force and not is_stale():
        return LIB
    return _compile(LIB, verbose, [])


def _compile(LIB, verbose, extra):
    cmd = [nvcc_path()] + NVCC_FLAGS + ['-Xcompiler', '-fPIC', '-shared', '-Xptxas', '-v' if verbose else '-O3',
           '-o', LIB] + extra + SOURCES + ['-ldl']
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError('nvcc failed')
    return LIB


if __name__ == '__main__':
    print(build(force=True, verbose='-v' in sys.argv, profile='--profile' in sys.argv, checks='--checks' in sys.argv))
