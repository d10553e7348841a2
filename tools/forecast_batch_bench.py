"""Cost of a pending-queue forecast on the batch path (``nhd_plan_batch_rounds``) on the BASELINE config-4 cluster
(65 536 nodes), next to ``nhd_plan_scenarios_rounds`` of the same pods as one scenario.

The cluster is config 4 with one more node group on a few of its GPU nodes (8 and 512); after the 4 096-pod solve the
pending set is one-GPU pods of the stream that request that group only, so each scan places at most one per such node
and the rest find no node.  64 and 4 096 pods over 1, 8 and 32 scans 30 s apart, without and with reasons, the two
calls alternating in one process; their outputs are asserted equal before anything is timed.  Prints per case the
device time of one call (kernels and device-side copies, summed per kernel from torch.profiler's CUDA activity, in a
run of its own), the host time per call (median of calls that end in the call's own wait), and the device time of a
plain ``nhd_plan_batch`` of the same pods: what the rounds cost beyond it is the advance kernels, the per-round solves
of the survivors and the record copy.  The card's name and power limit are read in the same run.

    python tools/forecast_batch_bench.py [--reps 5] [--json]
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
from forecast_bench import PERIOD, clocks, gpu_tail  # noqa: E402
from nhd_b200 import wire                           # noqa: E402
from nhd_b200.solver import Solver                  # noqa: E402


def grouped(recs, n_nodes):
    """``recs`` with a node group no node carries added to ``n_nodes`` of its GPU nodes, spread over the node order, and
    that group's bit."""
    bit = next(b for b in range(64) if not (int(np.bitwise_or.reduce(recs['group_mask'])) >> b) & 1)
    out = recs.copy()
    gpu_nodes = np.flatnonzero(recs['n_gpus'] > 0)
    out['group_mask'][gpu_nodes[::max(1, len(gpu_nodes) // n_nodes)][:n_nodes]] |= np.uint64(1 << bit)
    return out, bit


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch

    recs0, speed, pods, now = workload.make_workload(4)
    rows = []
    for n_nodes in (8, 512):
        recs, bit = grouped(recs0, n_nodes)
        s = Solver(speed)
        try:
            s.load_nodes(recs)
            s.solve_batch(pods, now)
            clock = float(now.max()) + 5.0
            for n_pods in (64, 4096):
                tail = gpu_tail(pods, n_pods)
                tail['group_mask'] = np.uint64(1 << bit)
                t0 = np.full(n_pods, clock)
                for scans in (1, 8, 32):
                    later = clocks(clock, scans - 1)
                    scen = [((), tail, t0, None, None, None, later)]
                    row = {'case': f'{n_nodes} nodes x {n_pods} pods x {scans} scans'}
                    for explain in (False, True):
                        got = s.plan_batch_rounds(tail, t0, later, explain=explain)
                        want = s.plan_scenarios(scen, explain=explain)[0]
                        assert want[0] == 0 and got[0].tobytes() == want[2].tobytes() and (got[1] == want[-1]).all()
                        assert not explain or (got[2] == want[3]).all()
                        reps = 1 if n_pods == 4096 else args.reps      # the one-warp call takes up to seconds here
                        key = 'reasons_' if explain else ''
                        for name, fn, r in (('batch', lambda: s.plan_batch_rounds(tail, t0, later, explain=explain), args.reps),
                                            ('scenario', lambda: s.plan_scenarios(scen, explain=explain), reps)):
                            dev, host, kern = timed(fn, r)
                            row[f'{key}{name}_device_ms'], row[f'{key}{name}_host_ms'] = round(dev, 4), round(host, 4)
                            row[f'{key}{name}_per_kernel_ms'] = kern
                    row['plan_batch_device_ms'] = round(timed(lambda: s.plan_batch(tail, t0), args.reps)[0], 4)
                    placed = got[1][got[0]['status'] == wire.PLACED]
                    row['placed_scan0'], row['placed_later'] = int((placed == 0).sum()), int((placed > 0).sum())
                    rows.append(row)
        finally:
            s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(recs0), 'period': PERIOD, 'reps': args.reps}
    try:
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs0)} nodes, scans {PERIOD} s apart")
        for r in rows:
            print(f"{r['case']:36s} batch {r['batch_device_ms']:.3f} ms device / {r['batch_host_ms']:.3f} ms host "
                  f"(reasons {r['reasons_batch_device_ms']:.3f} / {r['reasons_batch_host_ms']:.3f}); one scenario "
                  f"{r['scenario_device_ms']:.3f} / {r['scenario_host_ms']:.3f} (reasons {r['reasons_scenario_device_ms']:.3f} / "
                  f"{r['reasons_scenario_host_ms']:.3f}); plan_batch {r['plan_batch_device_ms']:.3f} ms device; placed "
                  f"{r['placed_scan0']} at scan 0, {r['placed_later']} later")
            print('    batch:    ' + ', '.join(f'{k} {v}' for k, v in r['batch_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
