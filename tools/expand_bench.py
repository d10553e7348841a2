"""Cost of cluster growth plans (``nhd_plan_scenarios_grown``) on the BASELINE config-4 cluster (65 536 nodes).

After the 4 096-pod solve of config 4, the pending tail is 64 of the batch's pods that request a node group no source
node carries, so every tail pod finds no node on the source cluster.  A scenario adds K nodes carrying that group
(copies of node 0's record before the solve), spread over the node order, and plans the tail.  Cases: 64 and 2 560
scenarios of K = 1, 8 and 64 added nodes, each without and with reasons (``why_counts``: many NO_CANDIDATE pods, so
this also measures the reasons' base pass with many failed pods).  Prints, per case, the device time of one call
(kernels and device-side copies, summed per kernel from torch.profiler's CUDA activity), the host time per call
(median) and the NO_CANDIDATE count of the call, next to the same scenarios without their additions.  The card's name
and power limit are read in the same run.

    python tools/expand_bench.py [--reps 5] [--json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import workload                                     # noqa: E402
from drains_bench import timed                      # noqa: E402
from nhd_b200 import wire                           # noqa: E402
from nhd_b200.solver import Solver                  # noqa: E402

TAIL = 64


def scenarios(recs, pods, clock, n_scen, k):
    """``n_scen`` scenarios of ``k`` added nodes each (scenario s: positions s * n / n_scen + 997 i, wrapped, sorted) and
    the tail that only they can take; and the same scenarios without additions."""
    n = len(recs)
    bit = next(b for b in range(64) if not (int(np.bitwise_or.reduce(recs['group_mask'])) >> b) & 1)
    cand = recs[[0]].copy()
    cand['group_mask'] = np.uint64(1 << bit)
    tail = pods[:TAIL].copy()
    tail['group_mask'] = np.uint64(1 << bit)
    clocks = np.full(len(tail), clock)
    grown, bare = [], []
    for s in range(n_scen):
        at = np.sort((s * n // n_scen + np.arange(k) * 997) % (n + 1)).astype('<i4')
        grown.append(((), tail, clocks, None, None, (at, np.repeat(cand, k))))
        bare.append(((), tail, clocks))
    return grown, bare


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch

    recs, speed, pods, now = workload.make_workload(4)
    s = Solver(speed)
    rows = []
    try:
        s.load_nodes(recs)
        s.solve_batch(pods, now)
        clock = float(now.max()) + 5.0
        for n_scen in (64, 2560):
            for k in (1, 8, 64):
                grown, bare = scenarios(recs, pods, clock, n_scen, k)
                dev, host, kern = timed(lambda: s.plan_scenarios(grown), args.reps)
                xdev, xhost, xkern = timed(lambda: s.plan_scenarios(grown, explain=True), args.reps)
                none = lambda res: sum(int((g[2]['status'] == wire.NO_CANDIDATE).sum()) for g in res)   # noqa: E731
                rows.append({'scenarios': n_scen, 'added_per_scenario': k, 'pods': n_scen * TAIL,
                             'call_device_ms': round(dev, 4), 'call_host_ms': round(host, 4), 'per_kernel_ms': kern,
                             'reasons_device_ms': round(xdev, 4), 'reasons_host_ms': round(xhost, 4),
                             'reasons_per_kernel_ms': xkern,
                             'no_candidate_without': none(s.plan_scenarios(bare)),
                             'no_candidate_with': none(s.plan_scenarios(grown))})
    finally:
        s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs), 'pending': TAIL, 'reps': args.reps}
    try:
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes, {TAIL} pending pods per scenario")
        for r in rows:
            print(f"{r['scenarios']:5d} scenarios x {r['added_per_scenario']:2d} added, {r['pods']:6d} pods: one call "
                  f"{r['call_device_ms']:.4f} ms device / {r['call_host_ms']:.4f} ms host; with reasons "
                  f"{r['reasons_device_ms']:.4f} ms device / {r['reasons_host_ms']:.4f} ms host; NO_CANDIDATE "
                  f"{r['no_candidate_without']} without the additions, {r['no_candidate_with']} with")
            print('    call:    ' + ', '.join(f'{k} {v}' for k, v in r['per_kernel_ms'].items()))
            print('    reasons: ' + ', '.join(f'{k} {v}' for k, v in r['reasons_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
