"""Freeze the UNMODIFIED reference's answer to "these running pods end at about these times: does the queue clear
then, or do I also need one more node like this one?" into tests/golden/live/departures.json.gz.

The sessions are make_release_golden.py's (``release_sessions``: pending queues longer than a scan places, and GPU pods
holding two RX/TX pairings on one NIC with CPU-only NIC pods pending).  Each session is played to its end state in
the reference; then, per case, the candidate nodes of the case are inserted into the reference scheduler's node dict
(make_expand_golden.py's ``add_nodes`` step: none, or one empty copy of the session's first node shape at the end),
and ``SCANS`` pending scans run ``period`` seconds apart with the case's deployed pods deleted between them
(make_release_golden.py's ``scan_steps``).  The schedules of a session are make_release_golden.py's delete plans and
no delete at all, each with and without the added node.  The file records, per case, the deletes (pod and seconds
after the first scan), the added nodes, the scan and node of every pending pod or None, and the reference's own reasons
at its last scan for the pods no scan placed.  The generator asserts that the file holds a pod that places only when
both an added node and a release are present, two schedules of one session with different outcomes, and a scan in
which two pods bind to one NIC whose counter a release drove negative.  Cases in which the reference raises or a
Kubernetes write fails are left out, as in the generators it reuses.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_departures_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_defrag_golden import _WriteFailures, pending_keys   # noqa: E402
from tests.golden.make_expand_golden import _AddNodes, _copy, grown_names   # noqa: E402
from tests.golden.make_plan_golden import mirror_session   # noqa: E402
from tests.golden.make_release_golden import SCANS, delete_plans, offset, release_sessions, scan_steps   # noqa: E402

PERIOD = 30.0


def departure_sessions():
    """``release_sessions()``: ``(name, script)``."""
    return release_sessions()


def added_node(script):
    """The addition of a session: one empty copy of its first node shape, at the end."""
    spec = next(s for s in script['nodes'] if s['hp_alloc'] > 0 and s.get('active', True))
    return [{'node': _copy(spec, 'added0'), 'before': None}]


def departure_session(item):
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
    rng = np.random.default_rng(sum(map(ord, name)) + 7)
    adds = added_node(script)
    out = []
    with _Attempts() as att, _WriteFailures() as failures, _AddNodes():
        start = len(_run(att, script))
        prefix_failures = failures.n
        for k, deletes in enumerate([[]] + delete_plans(deployed, PERIOD, rng)):
            for nodes in ([], adds):
                failures.n = 0
                att.log = []
                steps = script['steps'] + ([{'op': 'add_nodes', 'nodes': nodes}] if nodes else []) + \
                    scan_steps(PERIOD, deletes)
                try:
                    doc = H.run_reference(dict(script, steps=steps))
                except TypeError:               # the reference's own crash in SetPhysicalIdsFromMapping (Node.py:833)
                    continue
                log = list(att.log)
                if failures.n != prefix_failures:
                    continue
                assert list(doc['nodes']) == grown_names(names, nodes), name
                where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
                tries = {}
                for ns, pod, _ in log[start:]:
                    tries[(ns, pod)] = tries.get((ns, pod), 0) + 1
                placed = [None if where.get(f'{ns}/{pod}') is None else [tries[(ns, pod)] - 1, where[f'{ns}/{pod}']]
                          for ns, pod in pending]
                never = {p for p, q in zip(pending, placed) if q is None}
                out.append({'schedule': k, 'period': PERIOD, 'nodes': nodes, 'placed': placed,
                            'reasons': _last(log, start, never),
                            'departures': [[ns, pod, offset(gap, when, PERIOD)] for ns, pod, gap, when in deletes]})
    print(name, len(pending), 'pending,', len(deployed), 'deployed,', len(out), 'cases', flush=True)
    return {'name': name, 'pending': [list(p) for p in pending], 'deployed_on': on, 'cases': out}


def evidence(sessions):
    """Per kind, the cases that show it: a pod placed only with both the added node and the deletes of its schedule,
    two schedules of one session with different outcomes, and two pending pods bound by one scan to one node of a
    pairing session beyond the NICs its deletes freed (make_release_golden.py's ``evidence``)."""
    both = differ = cut = 0
    for s in sessions:
        by = {(c['schedule'], bool(c['nodes'])): c for c in s['cases']}
        outcomes = {}
        for (k, grown), c in by.items():
            outcomes.setdefault(grown, set()).add(str(c['placed']))
            alone, plain = by.get((k, False)), by.get((0, True))
            if grown and k and alone is not None and plain is not None:
                both += sum(p is not None and q is None and r is None
                            for p, q, r in zip(c['placed'], alone['placed'], plain['placed']))
            if s['name'].endswith('_pairing') and not grown:
                for scan in range(1, SCANS):
                    for nd in set(s['deployed_on'].values()):
                        freed = sum(s['deployed_on'][pod] == nd and off <= scan * c['period']
                                    for _, pod, off in c['departures'])
                        took = sum(p is not None and p[0] <= scan and p[1] == nd for p in c['placed'])
                        cut += took > freed
        differ += any(len(v) > 1 for v in outcomes.values())
    return both, differ, cut


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        res = pool.map(departure_session, departure_sessions(), chunksize=1)
    both, differ, cut = evidence(res)
    print(sum(len(r['cases']) for r in res), 'cases;', both, 'placed only with an added node and a release,', differ,
          'sessions whose schedules differ,', cut, 'cases with a shared negative NIC')
    assert both > 0 and differ > 0 and cut > 0, (both, differ, cut)
    live._save('departures', {'sessions': res})


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    main()
