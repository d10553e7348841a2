"""Freeze the UNMODIFIED reference's answer to "these running pods end at about these times: when does each pending pod
get in, and on which node?" into tests/golden/live/releases.json.gz.

The sessions are make_forecast_golden.py's ``queue_script`` sessions (more one-GPU pods pending than a scan places)
and ``pairing_script`` sessions: GPU pods deployed with two RX/TX pairings on one NIC each, then CPU-only NIC pods
pending that find every NIC taken.  Each session is played to its end state in the reference; then, per case, ``SCANS``
pending scans run ``period`` seconds apart, and between them deployed pods are deleted (a ``TRIAD_POD_DELETE`` watch
item and the pod's removal from Kubernetes) at chosen clocks: mid-gap, exactly at a scan's clock (before that scan),
and 10 s before a scan (inside ``MIN_BUSY_SECS``).  The clocks stay integral, so that a clock stepped in two parts equals the
clock stepped once.  The file records, per case, the deletes (pod and seconds after the first scan), the pods the
scans attempt, for each the scan that bound it and its node or None, and the reference's own reasons at its last scan
for every pod no scan placed.  The generator asserts that the file holds a pod that places only after a release, a GPU
pod that a release's busy stamp holds one scan longer, and a scan in which two pods bind to one NIC whose counter a
release drove negative.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_release_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_defrag_golden import _WriteFailures, pending_keys   # noqa: E402
from tests.golden.make_forecast_golden import queue_script   # noqa: E402
from tests.golden.make_plan_golden import mirror_session   # noqa: E402

SCANS = 4
PERIODS = (30.0, 10.0)
WHEN = ('mid', 'at', 'busy')            # where in its gap a delete lands


def pairing_script(seed):
    """Two GPU nodes with one NIC per NUMA node; one GPU pod per NIC, each with two RX/TX pairings on it, deployed one
    scan apart; then 3 to 5 CPU-only pods of one pairing each, which find every NIC taken."""
    from tests import scenarios as S
    rng = np.random.default_rng(seed)
    nodes = [S.make_node(f'n{i}', 2, 16, bool(rng.random() < 0.5), 1, [(0, 0, 0x10), (1, 1, 0x20)],
                         [('eth0', 100000, 0, 0x10), ('eth1', 100000, 1, 0x20)], hp_alloc=64, hp_free=64)
             for i in range(2)]
    steps = []
    for k in range(4):
        spec = S.make_pod([S.make_group([(10, 10), (10, 10)], 1, [k % 2], 0)], 1, False, 'NUMA', 0)
        steps += [{'op': 'add_pod', 'ns': 'ns0', 'name': f'g{k}', 'uid': f'ug{k}', 'fail': [], 'pod': spec},
                  {'op': 'idle'}, {'op': 'clock', 'dt': 31.0}]
    for k in range(int(rng.integers(3, 6))):
        spec = S.make_pod([S.make_group([(10, 10)], 1, [], 0)], 1, False, 'NUMA', 0)
        steps.append({'op': 'add_pod', 'ns': 'ns0', 'name': f'c{k}', 'uid': f'uc{k}', 'fail': [], 'pod': spec})
    steps += [{'op': 'idle'}, {'op': 'clock', 'dt': 5.0}]
    return {'nodes': nodes, 'min_busy_secs': 30.0, 'clock0': 1000.0, 'init': [], 'steps': steps, 'codec': 'json'}


def release_sessions():
    """``(name, script)``: the queue sessions and the pairing sessions."""
    return [(f'json{seed}_queue', queue_script(seed)) for seed in range(51, 59)] + \
        [(f'json{seed}_pairing', pairing_script(seed)) for seed in range(61, 65)]


def delete_plans(deployed, period, rng):
    """Deletes of deployed pods: ``[(ns, name, gap, when)]``, ``gap`` 1 .. SCANS - 1 the gap before that scan."""
    out = []
    for when in WHEN:
        pick = [deployed[i] for i in rng.permutation(len(deployed))[:min(len(deployed), 3)]]
        out.append([(ns, name, 1 + int(rng.integers(SCANS - 1)), when) for ns, name in pick])
    out.append([(ns, name, 1, 'mid') for ns, name in deployed])
    return out


def offset(gap, when, period):
    """Seconds after the first scan of a delete in gap ``gap`` (before scan ``gap``)."""
    into = {'mid': period / 2, 'at': period, 'busy': period - 10.0 if period > 10.0 else period / 2}[when]
    return (gap - 1) * period + into


def scan_steps(period, deletes):
    """``SCANS`` scans ``period`` apart with the deletes in their gaps (a delete exactly at a scan's clock before it)."""
    steps = [{'op': 'idle'}]
    for k in range(1, SCANS):
        t = 0.0
        for ns, name, gap, when in sorted((d for d in deletes if d[2] == k), key=lambda d: offset(d[2], d[3], period)):
            at = offset(gap, when, period) - (k - 1) * period
            if at > t:
                steps.append({'op': 'clock', 'dt': at - t})
                t = at
            steps += [{'op': 'watch', 'type': 'NHD_WATCH_TYPE_TRIAD_POD_DELETE', 'pod': {'ns': ns, 'name': name,
                                                                                         'uid': 'gone'}},
                      {'op': 'delete_pod', 'ns': ns, 'name': name}]
        if period > t:
            steps.append({'op': 'clock', 'dt': period - t})
        steps.append({'op': 'idle'})
    return steps


def release_session(item):
    from tests import helpers
    from tests import sched_harness as H
    from tests.golden.make_plan_reasons_golden import _Attempts, _last, _run
    name, script = item
    sched, _, _ = mirror_session(script, helpers.OracleSolver)
    try:
        pending = pending_keys(sched)
        deployed = [(ns, pod) for n in sched.nodes.values() for (pod, ns) in n.pod_info]
        on = {pod: nd for nd, n in sched.nodes.items() for (pod, ns) in n.pod_info}
    finally:
        sched.close()
    rng = np.random.default_rng(sum(map(ord, name)))
    out = []
    with _Attempts() as att, _WriteFailures() as failures:
        start = len(_run(att, script))
        prefix_failures = failures.n
        for period in PERIODS:
            for deletes in [[]] + delete_plans(deployed, period, rng):
                failures.n = 0
                att.log = []
                try:
                    doc = H.run_reference(dict(script, steps=script['steps'] + scan_steps(period, deletes)))
                except TypeError:               # the reference's own crash in SetPhysicalIdsFromMapping (Node.py:833)
                    continue
                log = list(att.log)
                if failures.n != prefix_failures:
                    continue
                where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
                tries = {}
                for ns, pod, _ in log[start:]:
                    tries[(ns, pod)] = tries.get((ns, pod), 0) + 1
                placed = [None if where.get(f'{ns}/{pod}') is None else [tries[(ns, pod)] - 1, where[f'{ns}/{pod}']]
                          for ns, pod in pending]
                never = {k for k, p in zip(pending, placed) if p is None}
                out.append({'period': period, 'placed': placed, 'reasons': _last(log, start, never),
                            'departures': [[ns, pod, offset(gap, when, period)] for ns, pod, gap, when in deletes]})
    print(name, len(pending), 'pending,', len(deployed), 'deployed,', len(out), 'cases', flush=True)
    return {'name': name, 'pending': [list(p) for p in pending], 'deployed_on': on, 'cases': out}


def evidence(sessions):
    """Per kind, the cases that show it: a pod placed only with the deletes, a pod placed later with them (a busy
    stamp), and two pending pods bound in one scan to one node of a pairing session beyond its free NICs."""
    after = held = cut = 0
    for s in sessions:
        base = {c['period']: c for c in s['cases'] if not c['departures']}
        for c in s['cases']:
            b = base.get(c['period'])
            if b is None or not c['departures']:
                continue
            for p, q in zip(c['placed'], b['placed']):
                after += p is not None and q is None
                held += p is not None and q is not None and p[0] > q[0]
            if s['name'].endswith('_pairing'):
                # every NIC of a pairing session is held by one GPU pod at first, and each pending pod takes one NIC:
                # more pending pods on a node by scan k than GPU pods released from it by then share a NIC
                for k in range(1, SCANS):
                    for nd in set(s['deployed_on'].values()):
                        freed = sum(s['deployed_on'][pod] == nd and off <= k * c['period']
                                    for _, pod, off in c['departures'])
                        took = sum(p is not None and p[0] <= k and p[1] == nd for p in c['placed'])
                        cut += took > freed
    return after, held, cut


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        res = pool.map(release_session, release_sessions(), chunksize=1)
    after, held, cut = evidence(res)
    print(sum(len(r['cases']) for r in res), 'cases;', after, 'placed only after a release,', held,
          'held longer by a busy stamp,', cut, 'cases with a cut')
    assert after > 0 and held > 0 and cut > 0, (after, held, cut)
    live._save('releases', {'sessions': res})


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    main()
