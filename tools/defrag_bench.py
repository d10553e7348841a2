"""Cost of defragmentation plans (``nhd_plan_scenarios_edited``) on the BASELINE config-4 cluster (65 536 nodes).

After the 4 096-pod solve of config 4, the pending set is that solve's NO_CANDIDATE pods, at most 64; config 4 places
every pod, so the first 64 pods of the batch stand in for it (they fit, so every scenario plans its whole tail).  A
node is drained and put back in service as ``NHDScheduler.PlanDefrag`` plans it: its pods re-planned at the drain's clock (5 s after
the last pod of the solve) with the node excluded, the node's record replaced by the one its pods' release leaves
behind (here the record before the solve, busy from the drain's clock), then the pending set at that clock + 30 s with
the exclusion lifted.  Three cases:
  * n-1: one call, one scenario per node holding pods;
  * racks: one call, 64 racks of 32 consecutive nodes (rack r = nodes 1024 r .. 1024 r + 31);
  * the same two sets as ``nhd_plan_scenarios`` of the drains alone (no edits, no lift, no pending tail): what the
    return-to-service phase adds;
  * each defrag set again with reasons (``nhd_plan_scenarios_explained``).
Prints, per case, the device time of one call (kernels and device-side copies, summed per kernel from torch.profiler's
CUDA activity) and the host time per call (median).  The card's name and power limit are read in the same run.

    python tools/defrag_bench.py [--reps 5] [--json]
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

CAP = 64


def scenario_sets(start, pods, node, clock, tail):
    def scenario(group):
        rows = np.sort(np.flatnonzero(np.isin(node, group)))
        recs = start[group].copy()
        recs['busy_time'] = clock
        drain = (group, pods[rows], np.full(len(rows), clock))
        return drain, (group, np.concatenate([pods[rows], tail]),
                       np.concatenate([np.full(len(rows), clock), np.full(len(tail), clock + 30.0)]), len(rows),
                       (group, recs))
    holding = np.unique(node[node >= 0])
    n1 = [scenario(np.asarray([n])) for n in holding]
    racks = [scenario(np.arange(r * 1024, r * 1024 + 32)) for r in range(64)]
    return {'n-1': n1, 'racks': racks}, len(tail)


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
        node = s.solve_batch(pods, now)['node']
        failed = np.flatnonzero(node < 0)[:CAP]
        tail = pods[failed] if len(failed) else pods[:CAP]    # config 4 places every pod: its first 64 stand in
        sets, n_tail = scenario_sets(recs, pods, node, float(now.max()) + 5.0, tail)
        for name, pairs in sets.items():
            drains = [d for d, _ in pairs]
            defrag = [f for _, f in pairs]
            dev, host, kern = timed(lambda: s.plan_scenarios(defrag), args.reps)
            ddev, dhost, dkern = timed(lambda: s.plan_scenarios(drains), args.reps)
            xdev, xhost, xkern = timed(lambda: s.plan_scenarios(defrag, explain=True), args.reps)
            rows.append({'set': name, 'scenarios': len(defrag), 'pods': int(sum(len(sc[1]) for sc in defrag)),
                         'call_device_ms': round(dev, 4), 'call_host_ms': round(host, 4), 'per_kernel_ms': kern,
                         'drains_only_device_ms': round(ddev, 4), 'drains_only_host_ms': round(dhost, 4),
                         'drains_only_per_kernel_ms': dkern, 'reasons_device_ms': round(xdev, 4),
                         'reasons_host_ms': round(xhost, 4), 'reasons_per_kernel_ms': xkern,
                         'no_candidate': sum(int((g[2]['status'] == wire.NO_CANDIDATE).sum()) for g in s.plan_scenarios(defrag))})
    finally:
        s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs), 'pending': n_tail, 'reps': args.reps}
    try:
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes, {n_tail} pending pods")
        for r in rows:
            print(f"{r['set']:6s} {r['scenarios']:5d} scenarios, {r['pods']:6d} pods: one call {r['call_device_ms']:.4f} ms "
                  f"device / {r['call_host_ms']:.4f} ms host; drains alone {r['drains_only_device_ms']:.4f} ms device / "
                  f"{r['drains_only_host_ms']:.4f} ms host")
            print('    call:   ' + ', '.join(f'{k} {v}' for k, v in r['per_kernel_ms'].items()))
            print('    drains: ' + ', '.join(f'{k} {v}' for k, v in r['drains_only_per_kernel_ms'].items()))
            print(f"    with reasons ({r['no_candidate']} NO_CANDIDATE pods): {r['reasons_device_ms']:.4f} ms device / "
                  f"{r['reasons_host_ms']:.4f} ms host")
            print('    reasons: ' + ', '.join(f'{k} {v}' for k, v in r['reasons_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
