"""A whole BASELINE configuration through the real kernels on the CPU-emulated device (tests/emu), every binding
and every final node record compared with the (multi-threaded) oracle.  Developer tool; needs no GPU.  The same
workloads as tests/test_gpu_full_size.py, which runs them on the GPU.

    python tools/emu_full_size.py 4                 # 65 536 nodes x 4 096 pods: ~4 s emulated device + ~75 s oracle on 8 cores
    python tools/emu_full_size.py 4 --wild          # the heterogeneous cluster (bench.py's extra), then a second batch
                                                    # on the same handle after an update of 1 024 nodes
    python tools/emu_full_size.py 4 --clock moving  # per-pod clocks 1 ms apart (bench.py's extra)
    python tools/emu_full_size.py 4 --clock jumps   # per-pod clocks with +31 s and -40 s steps (scenarios.jumping_clocks)
"""
import argparse, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
import build_emu_cuda
os.environ['NHD_B200_LIB']=build_emu_cuda.build()
os.environ['NHD_B200_ALLOW_EMULATED'] = '1'; os.environ['EMU_LANE_ORDER']='d'
import numpy as np
import workload
from nhd_b200.solver import Solver
from oracle import binding
from tests import helpers, ref_compare, scenarios

ap = argparse.ArgumentParser()
ap.add_argument('config', type=int)
ap.add_argument('--wild', action='store_true', help='the heterogeneous cluster of workload.make_cluster')
ap.add_argument('--clock', choices=('moving', 'jumps'), help='per-pod clocks instead of one clock for the batch')
args = ap.parse_args()
recs, speed, pods, now = workload.make_workload(args.config, wild=args.wild)
if args.clock == 'moving':
    now = now + 0.001 * np.arange(len(pods))
elif args.clock == 'jumps':
    now = scenarios.jumping_clocks(len(pods))
print(len(recs), len(pods), flush=True)


def compare(tag, ob, orecs, b, final):
    diff = helpers.first_binding_diff(ob, b)
    print(tag, 'bindings equal', diff is None, 'final equal', final.tobytes() == orecs.tobytes(),
          'placed', int((ob['status'] == 0).sum()), flush=True)
    if diff is not None:
        print('  first difference:', diff)
    if final.tobytes() != orecs.tobytes():
        print('  records:', ref_compare.diff_records(orecs, final)[:3])


s=Solver(speed); s.load_nodes(recs)
t0=time.time(); b=s.solve_batch(pods, now); print('emulated device', time.time()-t0,'s', flush=True)
final=s.read_nodes()
t0=time.time(); ob, orecs = binding.solve(recs, speed, pods, now, threads=os.cpu_count()); print('oracle mt', time.time()-t0,'s', flush=True)
compare('batch', ob, orecs, b, final)
if args.clock == 'jumps':
    print('backwards steps', int((np.diff(now) < 0).sum()),
          'GPU nodes with two or more GPU pods', len(scenarios.repeated_gpu_nodes(pods, ob)))
if args.wild:
    from tests.test_handle_session import static_key
    print('static descriptions', len({static_key(r) for r in recs}), 'NIC signatures', len(scenarios.nic_signatures(recs)))
    # the steady state: the same handle takes an update and a second batch a minute later
    idx, upd = scenarios.steady_state_update(recs, ob)
    pods2, now2 = workload.make_pods(args.config, n_pods=1024, seed=61)
    now2 = now2 + 60.0
    s.update_nodes(idx, upd)
    t0=time.time(); b2=s.solve_batch(pods2, now2); print('emulated device', time.time()-t0,'s', flush=True)
    final2=s.read_nodes()
    orecs[idx] = upd
    t0=time.time(); ob2, orecs2 = binding.solve(orecs, speed, pods2, now2, threads=os.cpu_count()); print('oracle mt', time.time()-t0,'s', flush=True)
    compare('second batch', ob2, orecs2, b2, final2)
s.close()
