import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, workload
from nhd_b200.solver import Solver
cfg = int(sys.argv[1]); cw = int(sys.argv[2])
recs, speed, pods, now = workload.make_workload(cfg)
for rep in range(6):
    s = Solver(speed, cpu_warps=cw)
    s.load_nodes(recs)
    try:
        b = s.solve_batch(pods, now)
        err = None
    except Exception as e:
        err = str(e)[:80]
    try:
        c = s.debug_counters()
        print('cfg', cfg, 'cw', cw, 'rep', rep, 'err', err, 'chk', [int(x) for x in c[56:62]], flush=True)
        if err:
            break
    except Exception as e:
        print('cfg', cfg, 'cw', cw, 'rep', rep, 'err', err, 'counters failed', str(e)[:60], flush=True)
        break
    s.close()
