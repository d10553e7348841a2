"""Cost of forecasting many departure schedules at once (``nhd_plan_scenarios_releases``) on the BASELINE config-4
cluster (65 536 nodes), next to ``nhd_plan_scenarios_rounds`` of the same scenarios without releases and next to a
loop of ``nhd_plan_batch_releases``, one call per schedule.

Config 4 with a node group only 64 of its GPU nodes carry; after its 4 096-pod solve, 64 and 2 560 schedules, each a
scenario of the same 128 pending one-GPU pods that request that group (twice the nodes that can take them) over 8
scans 30 s apart, with 1, 8 or 64 of the placed pods released over the gaps (round-robin over the rounds, mid-gap, one pairing per claimed NIC, the pods on the
group's nodes first, each schedule its own draw), with and without one added node (a fresh copy of a group node at
the end of the node order).  Prints per case the device time of one call (kernels and device-side copies, summed from
torch.profiler's CUDA activity), the host time per call (median), the same for the call without releases, and for
the loop of batch calls (64 schedules without an added node only: the batch path adds no nodes, and 2 560 of its calls
per case are left out to keep the run short).  The card's name and power limit are read in the same run.

    python tools/departures_bench.py [--reps 5] [--json]
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
from forecast_bench import PERIOD, clocks           # noqa: E402
from nhd_b200 import wire                           # noqa: E402
from nhd_b200.solver import Scenario, Solver        # noqa: E402
from releases_bench import releases                 # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch

    from tests.test_forecast_batch import config4_pending
    recs, speed, pods, now = workload.make_workload(4)
    rows = []
    s = Solver(speed)
    try:
        recs, tail_all = config4_pending(recs, pods, 128, 64)
        bit = int(tail_all['group_mask'][0])
        group_nodes = np.flatnonzero(recs['group_mask'] & np.uint64(bit))
        s.load_nodes(recs)
        b0 = s.solve_batch(pods, now)
        after = s.read_nodes()
        clock = float(now.max()) + 5.0
        t0 = np.full(len(tail_all), clock)
        later = clocks(clock, 8)
        add = ([len(recs)], recs[group_nodes[:1]])
        for n_sched in (64, 2560):
            for n_rel in (1, 8, 64):
                rel = [releases(b0, pods, after, n_rel, later, clock, 1, group_nodes, seed=k) for k in range(n_sched)]
                for grown in (False, True):
                    scs = [Scenario((), tail_all, t0, None, None, add if grown else None, later, r) for r in rel]
                    bare = [sc._replace(releases=None) for sc in scs]
                    got = s.plan_scenarios(scs)
                    base = s.plan_scenarios(bare)
                    row = {'case': f'{n_sched} schedules x {n_rel} releases' + (' + 1 node' if grown else '')}
                    runs = [('releases', lambda: s.plan_scenarios(scs)), ('rounds', lambda: s.plan_scenarios(bare))]
                    if n_sched == 64 and not grown:
                        runs.append(('batch_loop', lambda: [s.plan_batch_releases(tail_all, t0, later, *r) for r in rel]))
                    for name, fn in runs:
                        dev, host, kern = timed(fn, args.reps)
                        row[f'{name}_device_ms'], row[f'{name}_host_ms'] = round(dev, 4), round(host, 4)
                        row[f'{name}_per_kernel_ms'] = kern
                    for key, res in (('', got), ('rounds_', base)):
                        row[f'{key}placed_later'] = int(sum(((r[2]['status'] == wire.PLACED) & (r[3] >= 1)).sum()
                                                            for r in res))
                    rows.append(row)
    finally:
        s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs), 'period': PERIOD, 'reps': args.reps}
    try:
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes, 128 pending pods x 8 scans {PERIOD} s apart")
        for r in rows:
            loop = (f"; batch loop {r['batch_loop_device_ms']:.3f} / {r['batch_loop_host_ms']:.3f}"
                    if 'batch_loop_device_ms' in r else '; batch loop not measured')
            print(f"{r['case']:38s} releases {r['releases_device_ms']:.3f} ms device / {r['releases_host_ms']:.3f} ms "
                  f"host; without releases {r['rounds_device_ms']:.3f} / {r['rounds_host_ms']:.3f}{loop}; placed later "
                  f"{r['placed_later']} (without releases {r['rounds_placed_later']})")
            print('    releases: ' + ', '.join(f'{k} {v}' for k, v in r['releases_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
