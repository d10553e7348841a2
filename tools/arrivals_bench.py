"""Cost of forecasting pods created between the scans (``nhd_plan_scenarios_arrivals``) on the BASELINE config-4 cluster
(65 536 nodes), next to ``nhd_plan_scenarios_releases`` of the same pods given as pending at the start.

Config 4 with a node group only 64 of its GPU nodes carry; after its 4 096-pod solve, 64 and 2 560 timelines, each a
scenario of 8, 64 or 128 one-GPU pods that request that group (128: twice the group's nodes), created spread evenly
over the gaps before 8 later scans
30 s apart (each at its own clock inside its gap), with and without 8 departures of placed pods (round-robin over the gaps,
mid-gap, one pairing per claimed NIC, the pods on the group's nodes first, each timeline its own draw).  Prints per
case the device time of one call (kernels and device-side copies, summed from torch.profiler's CUDA activity) and the
host time per call (median), for the arrivals call and for the releases call with every pod pending at the start.  The
card's name and power limit are read in the same run.

    python tools/arrivals_bench.py [--reps 5] [--json]
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


def timeline(n, start, later):
    """``(arrive, now)`` of ``n`` pods created spread evenly over the gaps before ``later``, each at its own clock."""
    arrive = np.asarray([1 + q * len(later) // n for q in range(n)], dtype='<i4')
    now = np.zeros(n)
    for g in range(1, len(later) + 1):
        idx = np.flatnonzero(arrive == g)
        lo, hi = (start if g == 1 else later[g - 2]), later[g - 1]
        now[idx] = lo + (np.arange(len(idx)) + 1) / (len(idx) + 1) * (hi - lo)
    return arrive, now


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
        later = clocks(clock, 8)
        none = ([], np.zeros((0, wire.MAX_NICS), dtype='<i2'), np.zeros(0, dtype=wire.RELEASE_DTYPE))
        for n_tl in (64, 2560):
            for n_arr in (8, 64, 128):
                arrive, at = timeline(n_arr, clock, later)
                p = tail_all[:n_arr]
                for n_dep in (0, 8):
                    rel = [releases(b0, pods, after, n_dep, later, clock, 1, group_nodes, seed=k) if n_dep else none
                           for k in range(n_tl)]
                    scs = [Scenario((), p, at, None, None, None, later, r, arrive) for r in rel]
                    pending = [Scenario((), p, np.full(n_arr, clock), None, None, None, later, r) for r in rel]
                    got = s.plan_scenarios(scs)
                    base = s.plan_scenarios(pending)
                    row = {'case': f'{n_tl} timelines x {n_arr} arrivals' + (f' + {n_dep} departures' if n_dep else '')}
                    for name, fn in (('arrivals', lambda: s.plan_scenarios(scs)),
                                     ('pending', lambda: s.plan_scenarios(pending))):
                        dev, host, kern = timed(fn, args.reps)
                        row[f'{name}_device_ms'], row[f'{name}_host_ms'] = round(dev, 4), round(host, 4)
                        row[f'{name}_per_kernel_ms'] = kern
                    row['placed'] = int(sum((r[2]['status'] == wire.PLACED).sum() for r in got))
                    row['placed_on_creation'] = int(sum(((r[2]['status'] == wire.PLACED) & (r[4] == at)).sum()
                                                        for r in got))
                    row['pending_placed'] = int(sum((r[2]['status'] == wire.PLACED).sum() for r in base))
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
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes, 8 scans {PERIOD} s apart")
        for r in rows:
            print(f"{r['case']:42s} arrivals {r['arrivals_device_ms']:.3f} ms device / {r['arrivals_host_ms']:.3f} ms "
                  f"host; all pending {r['pending_device_ms']:.3f} / {r['pending_host_ms']:.3f}; placed "
                  f"{r['placed']}, {r['placed_on_creation']} on creation (all pending {r['pending_placed']})")
            print('    arrivals: ' + ', '.join(f'{k} {v}' for k, v in r['arrivals_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
