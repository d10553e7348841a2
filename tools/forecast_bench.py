"""Cost of pending-queue forecasts (``nhd_plan_scenarios_rounds``) on the BASELINE config-4 cluster (65 536 nodes).

After the 4 096-pod solve of config 4, the pending tail is one-GPU pods of the batch that request a node group no
source node carries; a scenario adds copies of the first GPU node's start record carrying that group, so only they
take the tail, a GPU node at most one GPU pod per scan: more pods than one scan can place.  Cases:
  * one scenario of 8 added nodes, 64 and 4 096 pending pods, over 1, 8 and 32 scans 30 s apart: one warp forecasting
    the whole pending set;
  * 64 and 2 560 scenarios of 1 and 8 added nodes and a 64-pod tail, over 8 scans.
Each case without and with reasons.  Prints, per case, the device time of one call (kernels and device-side copies,
summed per kernel from torch.profiler's CUDA activity), the host time per call (median), and how many pods the scans
placed at scan 0 and later.  The card's name and power limit are read in the same run.

    python tools/forecast_bench.py [--reps 5] [--json]
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

PERIOD = 30.0


def clocks(t0, k):
    """``k`` scan clocks after ``t0``, each the one before plus ``PERIOD``."""
    out, t = [], t0
    for _ in range(k):
        t = t + PERIOD
        out.append(t)
    return out


def gpu_tail(pods, n):
    one = pods[(pods['n_groups'] == 1) & (pods['groups']['n_gpus'][:, 0] == 1)]
    return np.resize(one, n).copy()


def grown_scenarios(recs, pods, clock, n_scen, k, scans, n_pods=64):
    n = len(recs)
    bit = next(b for b in range(64) if not (int(np.bitwise_or.reduce(recs['group_mask'])) >> b) & 1)
    cand = recs[[int(np.flatnonzero(recs['n_gpus'] > 0)[0])]].copy()
    cand['group_mask'] = np.uint64(1 << bit)
    tail = gpu_tail(pods, n_pods)
    tail['group_mask'] = np.uint64(1 << bit)
    later = clocks(clock, scans - 1)
    return [((), tail, np.full(len(tail), clock), None, None,
             (np.sort((s * n // n_scen + np.arange(k) * 997) % (n + 1)).astype('<i4'), np.repeat(cand, k)), later)
            for s in range(n_scen)]


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
        cases = []
        for n_pods in (64, 4096):
            for scans in (1, 8, 32):
                cases.append((f'1 scenario x {n_pods} pods x {scans} scans',
                              grown_scenarios(recs, pods, clock, 1, 8, scans, n_pods)))
        for n_scen in (64, 2560):
            for k in (1, 8):
                cases.append((f'{n_scen} scenarios x {k} added x 8 scans', grown_scenarios(recs, pods, clock, n_scen, k, 8)))
        for label, scens in cases:
            reps = 1 if '4096 pods' in label else args.reps      # one warp walking 4 096 pods per scan: seconds
            dev, host, kern = timed(lambda: s.plan_scenarios(scens), reps)
            xdev, xhost, xkern = timed(lambda: s.plan_scenarios(scens, explain=True), reps)
            res = s.plan_scenarios(scens)
            placed = [g[-1][g[2]['status'] == wire.PLACED] for g in res]
            rows.append({'case': label, 'pods': sum(len(sc[1]) for sc in scens),
                         'call_device_ms': round(dev, 4), 'call_host_ms': round(host, 4), 'per_kernel_ms': kern,
                         'reasons_device_ms': round(xdev, 4), 'reasons_host_ms': round(xhost, 4),
                         'reasons_per_kernel_ms': xkern,
                         'placed_scan0': int(sum((p == 0).sum() for p in placed)),
                         'placed_later': int(sum((p > 0).sum() for p in placed))})
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
            print(f"{r['case']:40s} {r['pods']:7d} pods: one call {r['call_device_ms']:.4f} ms device / "
                  f"{r['call_host_ms']:.4f} ms host; with reasons {r['reasons_device_ms']:.4f} ms device / "
                  f"{r['reasons_host_ms']:.4f} ms host; placed {r['placed_scan0']} at scan 0, {r['placed_later']} later")
            print('    call:    ' + ', '.join(f'{k} {v}' for k, v in r['per_kernel_ms'].items()))
            print('    reasons: ' + ', '.join(f'{k} {v}' for k, v in r['reasons_per_kernel_ms'].items()))


if __name__ == '__main__':
    main()
