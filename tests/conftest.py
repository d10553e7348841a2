import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


@pytest.fixture(scope='session')
def oracle_lib():
    from oracle import binding
    binding.build()
    return binding


@pytest.fixture(scope='session')
def emu():
    """g++ build of the product's scalar core (tests/emu), CPU-only logic check."""
    import ctypes
    import subprocess
    here = os.path.join(ROOT, 'tests', 'emu')
    so = os.path.join(here, '_emu.so')
    srcs = [os.path.join(here, 'nhd_emu.cpp'), os.path.join(ROOT, 'nhd_b200', 'csrc', 'nhd_core.cuh'),
            os.path.join(ROOT, 'include', 'nhd_b200.h')]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(['g++', '-O2', '-std=c++17', '-x', 'c++', '-fPIC', '-shared', '-ffp-contract=off',
                        '-o', so, srcs[0]], check=True)
    L = ctypes.CDLL(so)
    L.nhd_emu_tuple_hash.restype = ctypes.c_uint64
    L.nhd_emu_tuple_hash.argtypes = [ctypes.c_int] * 3
    return L
