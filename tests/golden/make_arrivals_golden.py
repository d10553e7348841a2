"""Freeze the UNMODIFIED reference's answer to "we submit these pods between the scans, and these running pods end: when
does each pod start, and on which node?" into tests/golden/live/arrivals.json.gz.

The sessions are make_release_golden.py's (``release_sessions``: the queue sessions of make_forecast_golden.py, more
one-GPU pods pending than a scan places, and the pairing sessions, CPU-only NIC pods pending that find every NIC
taken).  Each session is played to its end state in the reference; then, per case, the case's added node (none, or
make_departures_golden.py's copy of the session's first node shape) is inserted into the reference scheduler's node
dict, and ``SCANS`` pending scans run ``PERIOD`` seconds apart.  In the gaps, deployed pods are deleted (a
``TRIAD_POD_DELETE`` watch item and the pod's removal from Kubernetes, as make_release_golden.py does) and new pods are
created through the reference's own ``run()`` create branch: ``add_pod`` in Kubernetes, then a
``TRIAD_POD_CREATE`` watch item, which the reference answers with an attempt at that clock.  Events of one gap are
played by offset, a delete before a create at the same offset; a create exactly at a scan's offset comes before that
scan.  Each new pod copies the spec of a pending pod of the session (``like``).  Per delete plan (none and
make_release_golden.py's ``delete_plans``) the arrival sets are: one pod early in gap 1 and one early in gap 2 (inside
the busy window of the last scan), one late in gap 1 and one late in gap 2 (after it), one exactly at scans 1 and 2,
and one right before and one right after each delete (at its offset, so after it); the first set also with the added
node.  The file records, per case, the arrivals (key, ``like`` and offset), the deletes, the added nodes, for every
pending and arriving pod the offset of its placing attempt (its creation or a scan) and its node, or None, and the
reference's own reasons at its last attempt for the pods never placed.  A pending pod was attempted once by every scan
up to the one that bound it; an arrival once on its creation and then once by every scan from its gap's on.

The generator asserts that the file holds an arrival placed on creation; one that fails on creation and places at a
later scan; one placed on creation on the node an older pending pod got at the next scan in the same case without
arrivals, that pod then missing that scan; one placed on creation right after a delete on its node in its gap, whose
``like`` pod no scan places without deletes; and one that fails on creation and places at its gap's scan on a node a
delete later in its gap freed.  Cases in which the reference raises or a Kubernetes write fails are left out, as in the
generators it reuses.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_arrivals_golden.py
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_defrag_golden import _WriteFailures, pending_keys   # noqa: E402
from tests.golden.make_departures_golden import added_node   # noqa: E402
from tests.golden.make_expand_golden import _AddNodes, grown_names   # noqa: E402
from tests.golden.make_plan_golden import mirror_session   # noqa: E402
from tests.golden.make_release_golden import SCANS, delete_plans, offset, release_sessions   # noqa: E402

PERIOD = 30.0


def arrival_sessions():
    """``release_sessions()``: ``(name, script)``."""
    return release_sessions()


def arrival_sets(deletes, pending):
    """Per delete plan the arrival sets: ``[(like index, offset)]``, ``like`` an index into the pending pods."""
    n = len(pending)
    sets = [[(0, 1.0), (1 % n, PERIOD + 1.0)],                             # inside the busy window of the last scan
            [(0, PERIOD - 3.0), (1 % n, 2 * PERIOD - 3.0)],                # after it
            [(0, PERIOD), (1 % n, 2 * PERIOD)]]                            # exactly at scans 1 and 2
    around = []
    for k, (_, _, gap, when) in enumerate(deletes):
        at = offset(gap, when, PERIOD)
        if at - 2.0 > (gap - 1) * PERIOD:
            around.append((k % n, at - 2.0))
        around.append(((k + 1) % n, at))
    if around:
        sets.append(around)
    return sets


def scan_steps(deletes, arrivals):
    """``SCANS`` scans ``PERIOD`` apart; in each gap, by offset, the deletes (``(ns, name, gap, when)``) and the
    creates (``(ns, name, uid, spec, offset)``), a delete first at an equal offset."""
    steps = [{'op': 'idle'}]
    for k in range(1, SCANS):
        events = [(offset(g, w, PERIOD), 0, i, ('delete', ns, name)) for i, (ns, name, g, w) in enumerate(deletes)
                  if g == k]
        events += [(at, 1, i, ('create', ns, name, uid, spec)) for i, (ns, name, uid, spec, at) in enumerate(arrivals)
                   if (k - 1) * PERIOD < at <= k * PERIOD]
        t = 0.0
        for at, _, _, ev in sorted(events, key=lambda e: e[:3]):
            at -= (k - 1) * PERIOD
            if at > t:
                steps.append({'op': 'clock', 'dt': at - t})
                t = at
            if ev[0] == 'delete':
                steps += [{'op': 'watch', 'type': 'NHD_WATCH_TYPE_TRIAD_POD_DELETE',
                           'pod': {'ns': ev[1], 'name': ev[2], 'uid': 'gone'}},
                          {'op': 'delete_pod', 'ns': ev[1], 'name': ev[2]}]
            else:
                steps += [{'op': 'add_pod', 'ns': ev[1], 'name': ev[2], 'uid': ev[3], 'fail': [], 'pod': ev[4]},
                          {'op': 'watch', 'type': 'NHD_WATCH_TYPE_TRIAD_POD_CREATE',
                           'pod': {'ns': ev[1], 'name': ev[2], 'uid': ev[3]}}]
        if PERIOD > t:
            steps.append({'op': 'clock', 'dt': PERIOD - t})
        steps.append({'op': 'idle'})
    return steps


def _spec(script, ns, name):
    return next(st['pod'] for st in script['init'] + script['steps']
                if st.get('op') == 'add_pod' and (st['ns'], st['name']) == (ns, name))


def arrival_session(item):
    from tests import helpers
    from tests import sched_harness as H
    from tests.golden.make_plan_reasons_golden import _Attempts, _last, _run
    name, script = item
    sched, _, _ = mirror_session(script, helpers.OracleSolver)
    try:
        names = list(sched.nodes)
        pending = pending_keys(sched)
        deployed = [(ns, pod) for n in sched.nodes.values() for (pod, ns) in n.pod_info]
        on = {pod: nd for nd, n in sched.nodes.items() for (pod, ns) in n.pod_info}
    finally:
        sched.close()
    out = []
    if not pending:
        print(name, 'no pending pod', flush=True)
        return {'name': name, 'pending': [], 'deployed_on': on, 'cases': out}
    rng = np.random.default_rng(sum(map(ord, name)) + 11)
    adds = added_node(script)
    with _Attempts() as att, _WriteFailures() as failures, _AddNodes():
        start = len(_run(att, script))
        prefix_failures = failures.n
        for k, deletes in enumerate([[]] + delete_plans(deployed, PERIOD, rng)):
            for a, aset in enumerate([[]] + arrival_sets(deletes, pending)):
                for nodes in ([], adds) if (k, a) == (0, 1) else ([],):
                    arrivals = []
                    for j, (like, at) in enumerate(aset):
                        ns, pod = pending[like][:2]
                        arrivals.append((ns, f'new{j}', f'unew{j}', _spec(script, ns, pod), at))
                    failures.n = 0
                    att.log = []
                    steps = script['steps'] + ([{'op': 'add_nodes', 'nodes': nodes}] if nodes else []) + \
                        scan_steps(deletes, arrivals)
                    try:
                        doc = H.run_reference(dict(script, steps=steps))
                    except TypeError:           # the reference's own crash in SetPhysicalIdsFromMapping (Node.py:833)
                        continue
                    log = list(att.log)
                    if failures.n != prefix_failures:
                        continue
                    assert list(doc['nodes']) == grown_names(names, nodes), name
                    where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
                    tries = {}
                    for ns, pod, _ in log[start:]:
                        tries[(ns, pod)] = tries.get((ns, pod), 0) + 1
                    placed = []
                    for ns, pod in [tuple(p[:2]) for p in pending]:
                        nd = where.get(f'{ns}/{pod}')
                        placed.append(None if nd is None else [(tries[(ns, pod)] - 1) * PERIOD, nd])
                    for ns, pod, _, _, at in arrivals:
                        nd, n_try = where.get(f'{ns}/{pod}'), tries.get((ns, pod), 0)
                        assert n_try >= 1, (name, pod)                 # the create branch attempted it
                        gap = math.ceil(at / PERIOD)
                        placed.append(None if nd is None else [at if n_try == 1 else (gap + n_try - 2) * PERIOD, nd])
                    keys = [tuple(p[:2]) for p in pending] + [(ns, pod) for ns, pod, _, _, _ in arrivals]
                    never = {p for p, q in zip(keys, placed) if q is None}
                    out.append({'schedule': k, 'set': a, 'period': PERIOD, 'nodes': nodes, 'placed': placed,
                                'attempts': [tries.get((ns, pod), 0) for ns, pod, _, _, _ in arrivals],
                                'reasons': _last(log, start, never),
                                'arrivals': [[ns, pod, list(pending[like][:2]), at]
                                             for (ns, pod, _, _, at), (like, _) in zip(arrivals, aset)],
                                'departures': [[ns, pod, offset(gap, when, PERIOD)] for ns, pod, gap, when in deletes]})
    print(name, len(pending), 'pending,', len(deployed), 'deployed,', len(out), 'cases', flush=True)
    return {'name': name, 'pending': [list(p) for p in pending], 'deployed_on': on, 'cases': out}


def evidence(sessions):
    """Per kind, the arrivals that show it: placed on creation; failed on creation and placed at a later scan; placed
    on creation on the node an older pending pod got at the next scan without arrivals, that pod then missing that
    scan; placed on creation right after a delete on its node in its gap, its ``like`` pod never placed without
    deletes; failed on creation and placed at its gap's scan on a node a later delete of its gap freed."""
    created = later = took = freed = waited = 0
    for s in sessions:
        n_p = len(s['pending'])
        by = {(c['schedule'], c['set'], bool(c['nodes'])): c for c in s['cases']}
        for c in s['cases']:
            base = by.get((c['schedule'], 0, False))
            plain = by.get((0, 0, False))
            deps = [(s['deployed_on'][pod], off) for _, pod, off in c['departures']]
            for (ns, pod, like, at), p, n_try in zip(c['arrivals'], c['placed'][n_p:], c['attempts']):
                if p is None:
                    continue
                gap = math.ceil(at / PERIOD)
                if n_try == 1:
                    created += 1
                    scan = gap * PERIOD
                    if base is not None and not c['nodes']:
                        for q, b in zip(c['placed'][:n_p], base['placed'][:n_p]):
                            if b is not None and b[0] == scan and b[1] == p[1] and (q is None or q[0] > scan):
                                took += 1
                    if any(nd == p[1] and (gap - 1) * PERIOD < off <= at for nd, off in deps) and plain is not None:
                        li = [list(x[:2]) for x in s['pending']].index(list(like))
                        freed += plain['placed'][li] is None
                else:
                    later += 1
                    if p[0] == gap * PERIOD and any(nd == p[1] and at < off <= gap * PERIOD for nd, off in deps):
                        waited += 1
    return created, later, took, freed, waited


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        res = pool.map(arrival_session, arrival_sessions(), chunksize=1)
    ev = evidence(res)
    print(sum(len(r['cases']) for r in res), 'cases; arrivals placed on creation %d, later %d, taking an older pod\'s '
          'node %d, placed after a delete %d, waiting for a later delete %d' % ev)
    assert all(ev), ev
    live._save('arrivals', {'sessions': res})


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    main()
