"""Cost of a pending-queue forecast with running pods finishing (``nhd_plan_batch_releases``) on the BASELINE config-4
cluster (65 536 nodes), next to ``nhd_plan_batch_rounds`` of the same pods without releases.

Config 4 with a node group only 64 of its GPU nodes carry; after its 4 096-pod solve, 64 and 4 096 pending one-GPU
pods that request that group, over 8 and 32 scans 30 s apart, with 64 and 1 024 of the placed pods released over the
gaps (round-robin over the rounds, mid-gap, the pods on the group's nodes first).  One pairing per claimed
NIC brings each released NIC's counter to 0, so no cut happens, but the call still takes the segment path (a cut is
possible) every round: record copy, cut check and one host read per round.  A last case gives every released NIC two
pairings, so the next claims of those NICs cut their rounds.  Prints per case the device time of one call (kernels and
device-side copies, summed from torch.profiler's CUDA activity, in a run of its own), the host time per call (median),
the same for ``nhd_plan_batch_rounds`` without releases, and the pods each call places at a later scan.  The card's
name and power limit are read in the same run.

    python tools/releases_bench.py [--reps 5] [--json]
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
from nhd_b200.solver import Solver                  # noqa: E402
from tests.test_forecast_releases import release_of  # noqa: E402


def releases(b0, pods, after, n_rel, rounds, t0, pairings, group_nodes, seed=4):
    """``n_rel`` placed pods released round-robin over the gaps, mid-gap, those on the group's nodes first"""
    placed = np.flatnonzero(b0['status'] == wire.PLACED)
    on = np.isin(b0['node'][placed], group_nodes)
    rng = np.random.default_rng(seed)
    pick = np.concatenate([rng.permutation(placed[on]), rng.permutation(placed[~on])])[:n_rel]
    rels = []
    for k, i in enumerate(pick):
        rnd = 1 + k % len(rounds)
        lo = t0 if rnd == 1 else rounds[rnd - 2]
        rels.append(release_of(b0[i], pods[i], int(b0[i]['node']), rnd, lo + 0.5 * (rounds[rnd - 1] - lo), pairings))
    rels = np.array(sorted(rels, key=lambda x: (int(x['round']), float(x['clock']))), dtype=wire.RELEASE_DTYPE)
    tracked = sorted({int(x['node']) for x in rels})
    used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
    for q, node in enumerate(tracked):
        nn = int(after['n_nics'][node])
        used[q, :nn] = [int(after['nic_inuse'][node]) >> i & 1 for i in range(nn)]
    return tracked, used, rels


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
        recs, tail_all = config4_pending(recs, pods, 4096, 64)
        bit = int(tail_all['group_mask'][0])
        group_nodes = np.flatnonzero(recs['group_mask'] & np.uint64(bit))
        s.load_nodes(recs)
        b0 = s.solve_batch(pods, now)
        after = s.read_nodes()
        clock = float(now.max()) + 5.0
        cases = [(p, sc, r, 1) for p in (64, 4096) for sc in (8, 32) for r in (64, 1024)] + [(4096, 8, 1024, 2)]
        for n_pods, scans, n_rel, pairings in cases:
            tail = tail_all[:n_pods]
            t0 = np.full(n_pods, clock)
            later = clocks(clock, scans)
            tracked, used, rels = releases(b0, pods, after, n_rel, later, clock, pairings, group_nodes)
            got = s.plan_batch_releases(tail, t0, later, tracked, used, rels)
            base = s.plan_batch_rounds(tail, t0, later)
            row = {'case': f'{n_pods} pods x {scans} scans x {n_rel} releases' + (' (cuts)' if pairings > 1 else '')}
            for name, fn in (('releases', lambda: s.plan_batch_releases(tail, t0, later, tracked, used, rels)),
                             ('rounds', lambda: s.plan_batch_rounds(tail, t0, later))):
                dev, host, kern = timed(fn, args.reps)
                row[f'{name}_device_ms'], row[f'{name}_host_ms'] = round(dev, 4), round(host, 4)
                row[f'{name}_per_kernel_ms'] = kern
            for key, (out, rnd) in (('', got), ('rounds_', base)):
                placed = rnd[out['status'] == wire.PLACED]
                row[f'{key}placed_scan0'], row[f'{key}placed_later'] = int((placed == 0).sum()), int((placed > 0).sum())
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
        print(f"{info['gpu']} ({info['power_limit']}), {len(recs)} nodes, scans {PERIOD} s apart")
        for r in rows:
            print(f"{r['case']:44s} releases {r['releases_device_ms']:.3f} ms device / {r['releases_host_ms']:.3f} ms "
                  f"host; rounds {r['rounds_device_ms']:.3f} / {r['rounds_host_ms']:.3f}; placed later "
                  f"{r['placed_later']} (without releases {r['rounds_placed_later']})")
            print('    releases: ' + ', '.join(f'{k} {v}' for k, v in r['releases_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
