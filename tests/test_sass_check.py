"""The sweep's direct path compiles without local-memory or generic accesses (tools/sass_check.py; needs nvcc, no GPU).

A kernel parameter whose address escapes to an out-of-line call is copied to the stack, and every later field read
becomes a local load plus a generic access through the loaded pointer: extra round trips on the per-pod chain."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, ROOT)

NVCC = shutil.which('nvcc') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else None)
pytestmark = pytest.mark.skipif(NVCC is None, reason='needs nvcc')


def test_direct_path_ranges_found_in_source():
    import sass_check
    r = sass_check.direct_ranges()
    for name in sass_check.DIRECT_FUNCS + ('sweep_kernel pod loop 0', 'sweep_kernel pod loop 1'):
        lo, hi = r[name]
        assert 0 < lo < hi


def test_sweep_direct_path_has_no_local_or_generic_access(tmp_path):
    import sass_check
    cubin, log = sass_check.compile_cubin(str(tmp_path))
    sass = sass_check.disassemble(cubin)
    res = sass_check.resources(log)
    ranges = sass_check.direct_ranges()
    for short, mangled in sass_check.SWEEP.items():
        assert res[mangled]['spill_stores'] == 0 and res[mangled]['spill_loads'] == 0, (short, res[mangled])
        hits = sass_check.scan(sass, mangled, ranges)
        assert hits == [], (short, hits[:10])
