"""Cost of ``nhd_plan_scenarios`` on the BASELINE config-4 cluster (65 536 nodes), next to a loop of ``nhd_plan_batch``
over the same scenarios.

After the 4 096-pod solve of config 4 (so that the nodes hold pods), two scenario sets at one clock 5 s later:
  * N-1: one scenario per node holding pods, that node excluded and its pods (in batch order) re-planned;
  * racks: 64 racks of 32 consecutive nodes (rack r = nodes 1024 r .. 1024 r + 31), each excluded with its pods.
Prints, per set, the device time of one call (kernels and device-side copies, summed per kernel from torch.profiler's
CUDA activity), the host time per call (median), and the same two figures for the loop of ``nhd_plan_batch`` calls
answering the same scenarios one by one; then the same with reasons: ``nhd_plan_scenarios_explained`` and the loop of
``nhd_plan_batch(..., why_counts)``.  The card's name and power limit are read in the same run.

    python tools/drains_bench.py [--reps 5] [--json]
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


def scenario_sets(recs, pods, node, clock):
    order = np.argsort(node, kind='stable')
    holding, starts = np.unique(node[order], return_index=True)
    bounds = list(starts) + [len(order)]
    n1 = [([int(n)], pods[order[bounds[i]:bounds[i + 1]]], np.full(bounds[i + 1] - bounds[i], clock))
          for i, n in enumerate(holding) if n >= 0]
    racks = []
    for r in range(64):
        rack = np.arange(r * 1024, r * 1024 + 32)
        rows = np.sort(np.flatnonzero(np.isin(node, rack)))
        racks.append((rack, pods[rows], np.full(len(rows), clock)))
    return {'n-1': n1, 'racks': racks}


def timed(fn, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()                                                                       # warm-up
    host = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            host.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
    kern = {ev.key: ev.self_device_time_total / 1e3 / reps for ev in prof.key_averages() if ev.self_device_time_total > 0}
    return sum(kern.values()), statistics.median(host), {k: round(v, 4) for k, v in sorted(kern.items())}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--loop-reps', type=int, default=1)
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch

    recs, speed, pods, now = workload.make_workload(4)
    s = Solver(speed)
    rows = []
    try:
        s.load_nodes(recs)
        node = s.solve_batch(pods, now)['node']
        sets = scenario_sets(recs, pods, node, float(now.max()) + 5.0)
        for name, scens in sets.items():
            dev, host, kern = timed(lambda: s.plan_scenarios(scens), args.reps)

            def loop():
                for ex, p, c in scens:
                    s.plan_batch(p, c, exclude=ex)
            ldev, lhost, lkern = timed(loop, args.loop_reps)
            xdev, xhost, xkern = timed(lambda: s.plan_scenarios(scens, explain=True), args.reps)

            def xloop():
                for ex, p, c in scens:
                    s.plan_batch(p, c, exclude=ex, explain=True)
            xldev, xlhost, xlkern = timed(xloop, args.loop_reps)
            failed = sum(int((g[2]['status'] == wire.NO_CANDIDATE).sum()) for g in s.plan_scenarios(scens))
            rows.append({'set': name, 'scenarios': len(scens), 'pods': int(sum(len(p) for _, p, _ in scens)),
                         'no_candidate': failed,
                         'call_device_ms': round(dev, 4), 'call_host_ms': round(host, 4), 'per_kernel_ms': kern,
                         'loop_device_ms': round(ldev, 3), 'loop_host_ms': round(lhost, 3), 'loop_per_kernel_ms': lkern,
                         'reasons_call_device_ms': round(xdev, 4), 'reasons_call_host_ms': round(xhost, 4),
                         'reasons_per_kernel_ms': xkern, 'reasons_loop_device_ms': round(xldev, 3),
                         'reasons_loop_host_ms': round(xlhost, 3), 'reasons_loop_per_kernel_ms': xlkern})
    finally:
        s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs), 'reps': args.reps, 'loop_reps': args.loop_reps}
    try:
        import subprocess
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes")
        for r in rows:
            print(f"{r['set']:6s} {r['scenarios']:5d} scenarios, {r['pods']:5d} pods: one call {r['call_device_ms']:.4f} ms "
                  f"device / {r['call_host_ms']:.4f} ms host; loop of nhd_plan_batch {r['loop_device_ms']:.3f} ms device / "
                  f"{r['loop_host_ms']:.3f} ms host")
            print('    call: ' + ', '.join(f'{k} {v}' for k, v in r['per_kernel_ms'].items()))
            print('    loop: ' + ', '.join(f'{k} {v}' for k, v in r['loop_per_kernel_ms'].items()))
            print(f"    with reasons ({r['no_candidate']} NO_CANDIDATE pods): one call {r['reasons_call_device_ms']:.4f} ms "
                  f"device / {r['reasons_call_host_ms']:.4f} ms host; loop {r['reasons_loop_device_ms']:.3f} ms device / "
                  f"{r['reasons_loop_host_ms']:.3f} ms host")
            print('    call: ' + ', '.join(f'{k} {v}' for k, v in r['reasons_per_kernel_ms'].items()))
            print('    loop: ' + ', '.join(f'{k} {v}' for k, v in r['reasons_loop_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
