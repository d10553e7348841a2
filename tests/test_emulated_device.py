"""The CUDA kernels themselves on a machine without a GPU.

``tests/emu/cuda_emu.h`` is a small CPU emulation of the CUDA execution model (every thread of a block a
fiber, warp collectives as rendezvous that abort on divergent use, __syncthreads, atomics, mbarrier + bulk
copy); ``tests/emu/build_emu_cuda.py`` compiles the product's own sources — ``nhd_api.cu``,
``nhd_kernels.cuh``, ``nhd_core.cuh``, ``nhd_ingest.cpp`` — with g++ on top of it into
``tests/emu/_emu_cuda.so``, a library with the product's C-ABI.  This test runs every ``-m gpu`` test of the
repository (parity with the oracle, golden vectors, drop-in Matcher, scheduler sessions ...) in a child
process whose ``NHD_B200_LIB`` points at that library: the filter, the multi-warp sweep with its hand-off
protocol, resolve / core-id / commit kernels and the host side of the ABI all execute for real, on the CPU.

What this does and does not show: the *logic* of the kernels and the convergence rules of the warp
collectives (a lane of a mask that has exited, or lanes of one mask sitting in different collectives, abort
the run).  It says nothing about speed or the GPU memory model (one OS thread: sequentially consistent).
TEST INFRASTRUCTURE: the product library is built by nvcc only, and on the GPU box the same tests run on
the B200 (``NHD_B200_LIB`` unset)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def emu_cuda_lib():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
    try:
        import build_emu_cuda
    finally:
        sys.path.pop(0)
    return build_emu_cuda.build()


def _run_gpu_tests(lib, extra_env=None, select=None):
    env = dict(os.environ, NHD_B200_LIB=lib, NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d')
    env.update(extra_env or {})
    cmd = [sys.executable, '-m', 'pytest', 'tests', '-m', 'gpu', '-q', '-x', '-p', 'no:cacheprovider']
    if select:
        cmd += ['-k', select]
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_gpu_suite_passes_on_the_emulated_device(emu_cuda_lib, lane_order):
    """Between two collectives the lanes of a warp run in a fixed order: both orders must give the oracle's answers
    (a lane-0 update of a word the other lanes still have to read shows up as a divergence in one of them)."""
    # ascending: the whole -m gpu suite; descending: the parity tests proper and the limit cases (keeps the CPU suite
    # to a few minutes)
    res = _run_gpu_tests(emu_cuda_lib, extra_env={'EMU_LANE_ORDER': lane_order},
                         select=None if lane_order == 'a' else
                         'random_scenarios or constant_clock or clock_changes or edge_cases or gpu_limits')
    tail = (res.stdout + res.stderr)[-3000:]
    assert res.returncode == 0, tail
    last = [ln for ln in res.stdout.strip().splitlines() if 'passed' in ln][-1]
    assert 'failed' not in last and int(last.split()[0]) >= (90 if lane_order == 'a' else 35), last


@pytest.mark.parametrize('sched_seed', ['', '1', '2'], ids=['round_robin', 'shuffled1', 'shuffled2'])
def test_every_sweep_mode_against_the_oracle_random(emu_cuda_lib, oracle_lib, sched_seed):
    """tools/emu_fuzz.py: random clusters and pod streams, two batches per run, every sweep mode, with the
    warps scheduled round-robin or in a shuffled order that changes every round (lanes ascending)."""
    env = dict(os.environ, EMU_LANE_ORDER='a')
    if sched_seed:
        env['EMU_SCHED_SEED'] = sched_seed
    res = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'emu_fuzz.py'), '7000', '42'], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and ' 0 mismatches' in res.stdout, (res.stdout + res.stderr)[-2000:]


def test_driver_smoke_entry_point_on_the_emulated_device(emu_cuda_lib, oracle_lib):
    """``__graft_entry__.smoke()`` — the one small run on the GPU — end to end."""
    env = dict(os.environ, NHD_B200_LIB=emu_cuda_lib, NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d')
    res = subprocess.run([sys.executable, '-c', 'import __graft_entry__ as g; g.smoke()'], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and 'smoke ok' in res.stdout, (res.stdout + res.stderr)[-2000:]


def test_full_size_cluster_is_exact_on_the_emulated_device(emu_cuda_lib, oracle_lib):
    """BASELINE config 4 at its full 65 536 nodes: the first 384 pods of the stream through the real kernels, every
    binding and every final record against the oracle (``tools/emu_full_size.py`` does all 4 096 pods: equal)."""
    code = '''
import os, sys
import numpy as np
sys.path.insert(0, %r)
import workload
from nhd_b200.solver import Solver
from oracle import binding
from tests import helpers
recs, speed, pods, now = workload.make_workload(4)
pods, now = pods[:384], now[:384]
s = Solver(speed); s.load_nodes(recs)
b = s.solve_batch(pods, now); final = s.read_nodes(); s.close()
ob, orecs = binding.solve(recs, speed, pods, now, threads=os.cpu_count())
assert len(recs) == 65536 and helpers.binding_bytes_equal(ob, b), helpers.first_binding_diff(ob, b)
assert final.tobytes() == orecs.tobytes()
print('placed', int((ob['status'] == 0).sum()))
''' % ROOT
    env = dict(os.environ, NHD_B200_LIB=emu_cuda_lib, NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d')
    res = subprocess.run([sys.executable, '-c', code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, (res.stdout + res.stderr)[-2000:]
    assert res.stdout.split()[-2:] == ["placed", "384"]


RANK_CODE = '''
import ctypes, os, sys, time
import numpy as np
sys.path.insert(0, %(root)r)
ctypes.CDLL(%(nccl)r, mode=ctypes.RTLD_GLOBAL)            # soname libnccl.so.2: what the library resolves at run time
import workload
from nhd_b200.solver import Solver, nccl_unique_id
rank, world, tmp = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
idf = os.path.join(tmp, 'nccl_id')
if rank == 0:
    nid = nccl_unique_id()
    open(idf + '.tmp', 'wb').write(nid); os.rename(idf + '.tmp', idf)
else:
    t0 = time.time()
    while not os.path.exists(idf):
        time.sleep(0.02)
        assert time.time() - t0 < 60
    nid = open(idf, 'rb').read()
recs, speed, pods, now = workload.make_workload(%(config)d, n_nodes=%(nodes)d, n_pods=%(pods)d)
s = Solver(speed, rank=rank, world_size=world, nccl_id=nid)
s.load_nodes(recs)
b1 = s.solve_batch(pods[:len(pods) // 2], now[:len(pods) // 2])
b2 = s.solve_batch(pods[len(pods) // 2:], now[len(pods) // 2:])
np.save(os.path.join(tmp, 'bind%%d.npy' %% rank), np.concatenate([b1, b2]))
np.save(os.path.join(tmp, 'final%%d.npy' %% rank), s.read_nodes())
print('launches', s.timing()['n_launches'])
s.close()
'''


@pytest.mark.parametrize('world,config,min_pairs', [(2, 3, '1'), (4, 5, '1'), (2, 3, None)], ids=['2-cfg3-sharded', '4-cfg5-sharded', '2-cfg3-whole'])
def test_node_sharded_ranks_match_the_oracle(emu_cuda_lib, oracle_lib, tmp_path, world, config, min_pairs):
    """SURVEY 8e on the CPU: ``world`` processes, each with an emulated device and the full cluster, compute
    their shard of the bitmaps, exchange them with one all-gather (tests/emu/fake_nccl: shared memory instead
    of NVLink) and run the identical sweep — every rank must return the oracle's bindings and records."""
    import numpy as np
    import workload
    from tests import helpers
    nccl_dir = os.path.join(ROOT, 'tests', 'emu', 'fake_nccl')
    nccl = os.path.join(nccl_dir, 'libnccl.so.2')
    src = os.path.join(nccl_dir, 'fake_nccl.c')
    if not os.path.exists(nccl) or os.path.getmtime(nccl) < os.path.getmtime(src):
        subprocess.run(['gcc', '-O2', '-fPIC', '-shared', '-w', '-Wl,-soname,libnccl.so.2', '-o', nccl, src, '-lrt'], check=True)
    nodes, pods_n = 1800, 500                                       # 8 super-tiles of 256 nodes: uneven shards for 4 ranks
    code = RANK_CODE % dict(root=ROOT, nccl=nccl, config=config, nodes=nodes, pods=pods_n)
    env = dict(os.environ, NHD_B200_LIB=emu_cuda_lib, NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d')
    env.pop('NHD_SHARD_MIN_PAIRS', None)
    if min_pairs is not None:
        env['NHD_SHARD_MIN_PAIRS'] = min_pairs         # clusters this small are filtered whole by every rank otherwise
    procs = [subprocess.Popen([sys.executable, '-c', code, str(r), str(world), str(tmp_path)], cwd=ROOT, env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(world)]
    outs = [p.communicate(timeout=600) for p in procs]
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0, (o + e)[-2000:]
        # tables + filter + sweep + resolve + core ids + commit, and the all-gather + unpack only when sharded
        assert int(o.split('launches')[-1].split()[0]) == (8 if min_pairs is not None else 6), o[-200:]
    recs, speed, pods, now = workload.make_workload(config, n_nodes=nodes, n_pods=pods_n)
    ob, orecs = oracle_lib.solve(recs, speed, pods, now)
    for r in range(world):
        b = np.load(os.path.join(tmp_path, 'bind%d.npy' % r))
        final = np.load(os.path.join(tmp_path, 'final%d.npy' % r))
        assert helpers.binding_bytes_equal(ob, b), (r, helpers.first_binding_diff(ob, b))
        assert final.tobytes() == orecs.tobytes(), r
    assert (ob['status'] == 0).sum() > 100


def test_emulator_catches_divergent_collectives(emu_cuda_lib, tmp_path):
    """The emulation is only worth something if it refuses what the GPU leaves undefined."""
    src = tmp_path / 'bad.cpp'
    src.write_text('''
#include "cuda_emu.h"
__global__ void diverge(int* out) {
    int lane = threadIdx.x;
    if (lane & 1) out[lane] = __ballot_sync(0xFFFFFFFFu, 1);     /* odd lanes vote ...           */
    else __syncwarp();                                           /* ... even lanes only synchronise */
}
__global__ void gone(int* out) {
    int lane = threadIdx.x;
    if (lane == 7) return;                                       /* lane 7 leaves, the mask still names it */
    out[lane] = __shfl_sync(0xFFFFFFFFu, lane, 0);
}
__global__ void fine(int* out) {
    int lane = threadIdx.x & 31;
    unsigned m = __ballot_sync(0xFFFFFFFFu, lane < 5);
    out[threadIdx.x] = __shfl_sync(0xFFFFFFFFu, (int)m + lane, (lane + 1) & 31) + __shfl_up_sync(0xFFFFFFFFu, lane, 1);
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(out + 64, 1);
}
int main(int argc, char** argv) {
    static int buf[80];
    int* out = buf;
    if (argv[1][0] == 'd') EMU_LAUNCH(diverge, 1, 32, 0, 0, out);
    if (argv[1][0] == 'g') EMU_LAUNCH(gone, 1, 32, 0, 0, out);
    if (argv[1][0] == 'f') { EMU_LAUNCH(fine, 3, 64, 0, 0, out); printf("%d %d %d %d %d\\n", out[0], out[1], out[31], out[63], out[64]); }
    return 0;
}
''')
    exe = tmp_path / 'bad'
    emu = os.path.join(ROOT, 'tests', 'emu')
    subprocess.run(['g++', '-O1', '-std=c++17', '-I', emu, '-o', str(exe), str(src), os.path.join(emu, 'cuda_emu.cpp')],
                   check=True)
    ok = subprocess.run([str(exe), 'f'], capture_output=True, text=True)
    assert ok.returncode == 0 and ok.stdout.split() == ['32', '33', '61', '61', '3'], (ok.stdout, ok.stderr)
    d = subprocess.run([str(exe), 'd'], capture_output=True, text=True)
    assert d.returncode != 0 and 'divergent collectives' in d.stderr
    g = subprocess.run([str(exe), 'g'], capture_output=True, text=True)
    assert g.returncode != 0 and 'already left the kernel' in g.stderr
