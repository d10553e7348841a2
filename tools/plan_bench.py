"""Cost of ``nhd_plan_batch`` on the BASELINE config-4 cluster (65 536 nodes), next to the solve of the same pods.

For P = 64 and 4 096 pods of config 4's stream (the first P), from both sources (the mirror as loaded, and the snapshot
of it), with no excluded node and with 1 024 (a fixed random sample), with and without the per-reason counts.
Prints, per case, the device time of the plan per call (kernels and device-side copies, summed from torch.profiler's
CUDA activity), the host time per call (median; de-duplication, copies, launches and the wait included), and the
device time of the solve of those P pods (``nhd_last_timing``).

    python tools/plan_bench.py [--reps 10] [--json]
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
from nhd_b200.solver import Solver                  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--pods', default='64,4096')
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch
    from torch.profiler import ProfilerActivity, profile

    recs, speed, pods, now = workload.make_workload(4)
    exclude = np.sort(np.random.default_rng(4).choice(len(recs), 1024, replace=False))
    s = Solver(speed)
    rows = []
    try:
        for P in [int(x) for x in args.pods.split(',')]:
            s.load_nodes(recs)
            s.snapshot()
            s.solve_batch(pods[:P], now[:P])
            solve_ms = s.timing()['total_ms']
            s.restore()
            for source in ('mirror', 'snapshot'):
                for ex in ((), exclude):
                    for explain in (False, True):
                        kw = dict(source=source, exclude=ex, explain=explain)
                        s.plan_batch(pods[:P], now[:P], **kw)                      # warm-up
                        host = []
                        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                            for _ in range(args.reps):
                                t0 = time.perf_counter()
                                s.plan_batch(pods[:P], now[:P], **kw)
                                host.append((time.perf_counter() - t0) * 1e3)
                            torch.cuda.synchronize()
                        kern = {ev.key: ev.self_device_time_total / 1e3 / args.reps for ev in prof.key_averages()
                                if ev.self_device_time_total > 0}
                        dev = sum(kern.values())
                        kern = {k: round(v, 4) for k, v in kern.items()}
                        rows.append({'pods': P, 'source': source, 'excluded': len(ex), 'explain': explain,
                                     'solve_ms': round(solve_ms, 3), 'plan_device_ms': round(dev, 4),
                                     'plan_host_ms': round(statistics.median(host), 4), 'per_kernel_ms': kern})
    finally:
        s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs), 'reps': args.reps}
    try:
        import subprocess
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes, {args.reps} calls per case")
        for r in rows:
            print(f"P={r['pods']:5d} {r['source']:8s} excluded={r['excluded']:4d} explain={int(r['explain'])}: "
                  f"plan {r['plan_device_ms']:.4f} ms device / {r['plan_host_ms']:.4f} ms host per call; "
                  f"solve of the same pods {r['solve_ms']:.3f} ms")
            print('    ' + ', '.join(f'{k} {v}' for k, v in r['per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
