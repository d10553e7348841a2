"""Cost of ``nhd_explain_batch`` on the BASELINE config-4 cluster (65 536 nodes) with F = 1, 64 and 4 096 pods that find
no node.

The batch is config 4's 4 096 pods (all placed) followed by 4 096 pods no node can take
(``tests.explain_scenarios.oversized_tail``); for each F the shortest prefix of that stream with F NO_CANDIDATE pods is solved once (snapshot -> solve) and
``explain_batch`` is then called repeatedly on it.  Prints, per F, the device time of the explanation kernels per call
(their durations summed from torch.profiler's CUDA activity), the host time per call (launches, the synchronisation
and the copy of the counts included) and both per failed pod, next to the solve's own device time (``nhd_last_timing``).

    python tools/explain_bench.py [--reps 20] [--json]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import workload                                     # noqa: E402
from nhd_b200 import wire                           # noqa: E402
from nhd_b200.solver import Solver                  # noqa: E402
from tests.explain_scenarios import oversized_tail  # noqa: E402


def _kernel_ms(prof):
    """Summed device time (ms) of the explanation kernels in a torch.profiler trace."""
    return sum(ev.self_device_time_total for ev in prof.key_averages() if 'explain_' in ev.key) / 1e3


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--fails', default='1,64,4096')
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch
    from torch.profiler import ProfilerActivity, profile

    recs, speed, pods, now = workload.make_workload(4)
    stream = np.concatenate([pods, oversized_tail(pods, len(pods))])
    clock = np.concatenate([now, np.full(len(pods), now[-1])])
    s = Solver(speed)
    rows = []
    try:
        s.load_nodes(recs)
        s.snapshot()
        status = s.solve_batch(stream, clock)['status']
        cum = np.cumsum(status == wire.NO_CANDIDATE)
        for F in [int(x) for x in args.fails.split(',')]:
            if cum[-1] < F:
                raise SystemExit(f'the stream has only {int(cum[-1])} NO_CANDIDATE pods')
            m = int(np.searchsorted(cum, F)) + 1                     # shortest prefix with F failures
            s.restore()
            s.snapshot()
            b = s.solve_batch(stream[:m], clock[:m])
            solve_ms = s.timing()['total_ms']
            assert int((b['status'] == wire.NO_CANDIDATE).sum()) == F
            counts = s.explain_batch()                               # warm-up (first launch loads the kernels)
            assert (counts[b['status'] == wire.NO_CANDIDATE].sum(axis=1) == len(recs)).all()
            host = []
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    s.explain_batch()
                    host.append((time.perf_counter() - t0) * 1e3)
                torch.cuda.synchronize()
            dev = _kernel_ms(prof) / args.reps
            host_ms = statistics.median(host)
            rows.append({'failed_pods': F, 'batch_pods': m, 'solve_ms': round(solve_ms, 3),
                         'explain_device_ms': round(dev, 3), 'explain_host_ms': round(host_ms, 3),
                         'device_ms_per_failed_pod': round(dev / F, 4), 'host_ms_per_failed_pod': round(host_ms / F, 4)})
    finally:
        s.close()
    if args.json:
        print(json.dumps({'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs), 'rows': rows}))
    else:
        print(f'{torch.cuda.get_device_name(0)}, {len(recs)} nodes')
        for r in rows:
            print(f"F={r['failed_pods']:5d} (batch {r['batch_pods']:5d}, solve {r['solve_ms']:.3f} ms): explain "
                  f"{r['explain_device_ms']:.3f} ms device / {r['explain_host_ms']:.3f} ms host per call, "
                  f"{r['device_ms_per_failed_pod']:.4f} / {r['host_ms_per_failed_pod']:.4f} ms per failed pod")


if __name__ == '__main__':
    main()
