"""Cost of forecasting one large timeline with pods created between the scans on the batch path
(``nhd_plan_batch_arrivals``) on the BASELINE config-4 cluster (65 536 nodes), next to ``nhd_plan_scenarios_arrivals``
of the same timeline as one scenario (one warp) and ``nhd_plan_batch_releases`` of the same pods given as pending at
the start.

Config 4 with a node group that 8 or 512 of its GPU nodes carry; after its 4 096-pod solve, 64 or 4 096 one-GPU pods
that request that group arrive as one burst at one clock in gap 1, or spread evenly over the gaps before 8 or 32 later
scans 30 s apart (each at its own clock), with 0, 64 or 1 024 departures of placed pods (round-robin over the gaps,
mid-gap, the pods on the group's nodes first).  One case also moves every departure to a random clock inside its gap,
so that releases interleave with the arrivals and each gap is solved as many small runs.  The outputs of the three
calls are compared before anything is timed: the batch and the scenario calls byte for byte (bindings, rounds, clocks).
Prints per case the device time of one call (kernels and device-side copies, summed from torch.profiler's CUDA
activity) and the host time per call (median).  A scenario call whose first run takes more than ``--limit`` seconds
is not timed and reads "not measured".  The card's name and power limit are read in the same run.

    python tools/batch_arrivals_bench.py [--reps 3] [--limit 10] [--json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import workload                                     # noqa: E402
from arrivals_bench import timeline                 # noqa: E402
from drains_bench import timed                      # noqa: E402
from forecast_bench import PERIOD, clocks           # noqa: E402
from nhd_b200 import wire                           # noqa: E402
from nhd_b200.solver import Scenario, Solver        # noqa: E402
from releases_bench import releases                 # noqa: E402

CASES = [  # (group nodes, arrivals, scans, departures, shape)
    (8, 64, 8, 0, 'burst'), (8, 4096, 8, 0, 'burst'), (8, 64, 8, 0, 'spread'), (8, 4096, 8, 0, 'spread'),
    (8, 4096, 8, 64, 'spread'), (8, 4096, 32, 64, 'spread'), (8, 4096, 8, 1024, 'interleaved'),
    (512, 64, 8, 0, 'burst'), (512, 4096, 8, 0, 'burst'), (512, 4096, 8, 0, 'spread'), (512, 4096, 32, 0, 'spread'),
    (512, 4096, 8, 64, 'spread'), (512, 4096, 8, 1024, 'spread'), (512, 4096, 8, 1024, 'interleaved'),
]


def interleave(rel, start, later, rng):
    """``rel`` with each release moved to a random clock inside its gap, array order = clock order."""
    tracked, used, rels = rel
    rels = rels.copy()
    for k in range(len(rels)):
        g = int(rels[k]['round'])
        lo, hi = (start if g == 1 else later[g - 2]), later[g - 1]
        rels[k]['clock'] = lo + rng.random() * (hi - lo)
    return tracked, used, rels[np.argsort(rels['clock'], kind='stable')]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--limit', type=float, default=10.0)
    ap.add_argument('--json', action='store_true')
    args = ap.parse_args(argv)
    import torch

    from tests.test_forecast_batch import config4_pending
    base_recs, speed, pods, now = workload.make_workload(4)
    rows = []
    rng = np.random.default_rng(18)
    none = ([], np.zeros((0, wire.MAX_NICS), dtype='<i2'), np.zeros(0, dtype=wire.RELEASE_DTYPE))
    for n_group in (8, 512):
        recs, tail_all = config4_pending(base_recs, pods, 4096, n_group)
        bit = int(tail_all['group_mask'][0])
        group_nodes = np.flatnonzero(recs['group_mask'] & np.uint64(bit))
        s = Solver(speed)
        try:
            s.load_nodes(recs)
            b0 = s.solve_batch(pods, now)
            after = s.read_nodes()
            clock = float(now.max()) + 5.0
            for g, n_arr, n_scans, n_dep, shape in CASES:
                if g != n_group:
                    continue
                later = clocks(clock, n_scans)
                p = tail_all[:n_arr]
                if shape == 'burst':
                    arrive, at = np.ones(n_arr, dtype='<i4'), np.full(n_arr, clock + 1.0)
                else:
                    arrive, at = timeline(n_arr, clock, later)
                rel = releases(b0, pods, after, n_dep, later, clock, 1, group_nodes) if n_dep else none
                if shape == 'interleaved':
                    rel = interleave(rel, clock, later, rng)
                start = np.full(n_arr, clock)
                sc = Scenario((), p, at, None, None, None, later, rel, arrive)

                def batch():
                    return s.plan_batch_arrivals(p, at, later, *rel, arrive)

                def pending():
                    return s.plan_batch_releases(p, start, later, *rel)

                def scenario():
                    return s.plan_scenarios([sc])
                b, rnd, clk = batch()
                t0 = time.perf_counter()
                (code, _, sb, srnd, sclk), = scenario()
                first = time.perf_counter() - t0
                assert code == 0 and sb.tobytes() == b.tobytes() and (srnd == rnd).all() and \
                    sclk.tobytes() == clk.tobytes(), (g, n_arr, n_scans, n_dep, shape)
                pending()
                row = {'case': f'{n_arr} {shape} arrivals, {n_scans} scans, {n_dep} departures, {g} group nodes',
                       'placed': int((b['status'] == wire.PLACED).sum()),
                       'placed_on_creation': int(((b['status'] == wire.PLACED) & (clk == at)).sum()),
                       'pending_placed': int((pending()[0]['status'] == wire.PLACED).sum())}
                for name, fn in (('batch', batch), ('pending', pending), ('scenario', scenario)):
                    if name == 'scenario' and first > args.limit:
                        row['scenario_device_ms'] = row['scenario_host_ms'] = 'not measured'
                        row['scenario_first_run_s'] = round(first, 2)
                        continue
                    dev, host, kern = timed(fn, args.reps)
                    row[f'{name}_device_ms'], row[f'{name}_host_ms'] = round(dev, 4), round(host, 4)
                    if name == 'batch':
                        row['batch_per_kernel_ms'] = kern
                rows.append(row)
                if not args.json:
                    print(row, flush=True)
        finally:
            s.close()
    info = {'gpu': torch.cuda.get_device_name(0), 'nodes': len(base_recs), 'period': PERIOD, 'reps': args.reps}
    try:
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                # the tool is optional for the measurement itself
        info['power_limit'] = 'unknown'
    if args.json:
        print(json.dumps(dict(info, rows=rows)))
    else:
        print(f"{info['gpu']} ({info['power_limit']}), {len(base_recs)} nodes, scans {PERIOD} s apart")
        for r in rows:
            print(f"{r['case']:64s} batch {r['batch_device_ms']} ms device / {r['batch_host_ms']} ms host; "
                  f"one warp {r['scenario_device_ms']} / {r['scenario_host_ms']}; all pending "
                  f"{r['pending_device_ms']} / {r['pending_host_ms']}; placed {r['placed']} "
                  f"({r['placed_on_creation']} on creation; all pending {r['pending_placed']})")


if __name__ == '__main__':
    main()
