"""bench.py's own arm on the CPU-emulated device of tests/emu with a stand-in `torch`: a dry run of the script's control
flow before it is spent on the GPU.  The numbers it prints describe the emulation, not the GPU.  Developer tool.

    python tools/bench_dry_run.py --steps 2 --warmup 3 --cpu-sample-pods 16             (N = 1, full-size workload)
    python tools/bench_dry_run.py --world 2 --small --steps 2 --warmup 3                 (2 ranks: stand-ins for
        torch.distributed (files in a temporary directory) and NCCL (tests/emu/fake_nccl), small clusters)
"""
import os, sys, types, runpy, subprocess, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
import numpy as np

argv = sys.argv[1:]
world = 1
if '--world' in argv:
    i = argv.index('--world'); world = int(argv[i + 1]); del argv[i:i + 2]
small = '--small' in argv
if small:
    argv.remove('--small')

if world > 1 and 'RANK' not in os.environ:
    # parent: one child per rank, then show rank 0's line
    import build_emu_cuda
    lib = build_emu_cuda.build()
    nccl_dir = os.path.join(ROOT, 'tests', 'emu', 'fake_nccl')
    nccl = os.path.join(nccl_dir, 'libnccl.so.2')
    if not os.path.exists(nccl):
        subprocess.run(['gcc', '-O2', '-fPIC', '-shared', '-w', '-Wl,-soname,libnccl.so.2', '-o', nccl,
                        os.path.join(nccl_dir, 'fake_nccl.c'), '-lrt'], check=True)
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        for r in range(world):
            env = dict(os.environ, RANK=str(r), LOCAL_RANK='0', WORLD_SIZE=str(world), DRY_TMP=tmp, DRY_NCCL=nccl)   # one emulated device per process
            procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), '--world', str(world)] + (['--small'] if small else []) +
                                          argv + ['--gpus', str(world)], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=3000) for p in procs]
        for r, (p, (o, e)) in enumerate(zip(procs, outs)):
            print(f'--- rank {r}: rc {p.returncode}\n{o[-3000:]}{e[-1500:] if p.returncode else ""}')
        sys.exit(max(p.returncode for p in procs))

import build_emu_cuda
os.environ['NHD_B200_LIB'] = build_emu_cuda.build()
os.environ['NHD_B200_ALLOW_EMULATED'] = '1'; os.environ['EMU_LANE_ORDER'] = 'd'
if world > 1:
    import ctypes
    ctypes.CDLL(os.environ['DRY_NCCL'], mode=ctypes.RTLD_GLOBAL)       # soname libnccl.so.2: what the library resolves at run time


class T:
    """the few tensor operations bench.py uses, on numpy"""
    def __init__(self, a): self.a = np.array(a)
    def zero_(self): return self
    def copy_(self, o): self.a[...] = o.a; return self
    def cpu(self): return self
    def cuda(self): return self
    def clone(self): return T(self.a.copy())
    def numpy(self): return self.a
    def item(self): return self.a.reshape(-1)[0].item()
    def all(self): return bool(self.a.all())
    def __eq__(self, o): return T(self.a == o.a)


torch = types.ModuleType('torch')
torch.uint8, torch.float64 = np.uint8, np.float64
torch.empty = lambda n, dtype=None, device=None: T(np.zeros(1, dtype=np.uint8))
torch.zeros = lambda n, dtype=None, device=None: T(np.zeros(n, dtype=dtype or np.float64))
torch.tensor = lambda v, dtype=None, device=None: T(np.array(v, dtype=dtype))
torch.frombuffer = lambda b, dtype=None: T(np.frombuffer(bytes(b), dtype=dtype).copy())
torch.cuda = types.SimpleNamespace(is_available=lambda: True, set_device=lambda d: None, synchronize=lambda: None,
                                   get_device_properties=lambda d: types.SimpleNamespace(uuid='none'))
torch.device = lambda *a: None
dist = types.ModuleType('torch.distributed')
rank = int(os.environ.get('RANK', '0'))
seq = [0]


def exchange(arr):
    """every rank's array, in rank order (files in DRY_TMP)"""
    tmp = os.environ['DRY_TMP']; k = seq[0]; seq[0] += 1
    np.save(os.path.join(tmp, f'c{k}_{rank}.tmp.npy'), arr)
    os.rename(os.path.join(tmp, f'c{k}_{rank}.tmp.npy'), os.path.join(tmp, f'c{k}_{rank}.npy'))
    out = []
    for r in range(world):
        f = os.path.join(tmp, f'c{k}_{r}.npy'); t0 = time.time()
        while not os.path.exists(f):
            time.sleep(0.005)
            assert time.time() - t0 < 1200, 'a rank is missing from a collective'
        out.append(np.load(f))
    return out


dist.ReduceOp = types.SimpleNamespace(MAX='max', SUM='sum')
dist.init_process_group = lambda *a, **k: None
dist.destroy_process_group = lambda: None
dist.barrier = lambda: exchange(np.zeros(1)) and None


def broadcast(t, src): t.a[...] = exchange(t.a)[src]


def all_reduce(t, op='sum'):
    parts = exchange(t.a)
    t.a[...] = np.max(parts, axis=0) if op == 'max' else np.sum(parts, axis=0)


dist.broadcast, dist.all_reduce = broadcast, all_reduce
torch.distributed = dist
sys.modules['torch'] = torch; sys.modules['torch.distributed'] = dist
if small:
    import workload
    full = workload.make_workload
    workload.make_workload = lambda cfg, n_nodes=None, n_pods=None, **kw: full(cfg, n_nodes or 4096, n_pods or 256, **kw)
sys.argv = ['bench.py'] + argv
os.chdir(ROOT)
runpy.run_path(os.path.join(ROOT, 'bench.py'), run_name='__main__')
