"""Freeze the UNMODIFIED reference's answer to "where would this pod go on its own?" into tests/golden/live/query.json.gz.

For every pod of a stream and each of a few states along that stream, the reference's ``Matcher.FindNode`` on that
state (after ``InitialNodeFilter``) and, on a deep copy of the nodes, ``SetBusy`` + ``SetPhysicalIdsFromMapping`` +
``ClaimPodNICResources`` (``ref_loader.attempt_scheduling``): node, mapping, core ids, GPU indices and claimed NICs,
``(None,)``, or the ``IndexError`` / ``TypeError`` of a failed assignment.  The states are the stream's start and the
cluster after its first third and its first two thirds were scheduled by the reference, one pod after the other.
Streams: the four ``oracle_scenarios`` flavours of make_live_golden.py, ``tests.explain_scenarios.explain_scenarios()``
and ``scenarios.limit_scenarios()`` (pre-used cores and NICs applied to the reference's node objects; the cases with
thousands of nodes are left out, their deep copies per pod would take hours).

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_query_golden.py
"""
import contextlib
import copy
import io
import logging
import os
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402

MAX_LIMIT_NODES = 512


def query_streams():
    """(name, scenarios) of the frozen comparison, shared with tests/test_query.py."""
    from tests import scenarios
    from tests.explain_scenarios import explain_scenarios
    out = [(f, live.oracle_scenarios(f)) for f in ('mixed', 'wild', 'vf', 'big')]
    out.append(('explain', explain_scenarios()))
    out.append(('limits', [s for s in scenarios.limit_scenarios() if len(s['nodes']) <= MAX_LIMIT_NODES]))
    return out


def query_states(scn):
    """Number of pods of the stream scheduled before each frozen state."""
    n = len(scn['pods'])
    return sorted({0, n // 3, (2 * n) // 3})


def _preuse(scn, nodes):
    for i, node in enumerate(nodes.values()):
        for c in scn.get('used', {}).get(i, ()):
            node.cores[c].used = True
        m = scn.get('nic_inuse', {}).get(i, 0)
        for k, nic in enumerate(node.nics):
            if (m >> k) & 1:
                nic.pods_used = max(nic.pods_used, 1)


def _outcome(names, nodes, r, top):
    from tests import scenarios
    o = {'status': r['status']}
    if r['status'] != 'none':
        node = nodes[r['node']]
        o['node'] = names.index(r['node'])
        m = r['mapping']
        o['mapping'] = {'gpu': list(m['gpu']), 'cpu': list(m['cpu']), 'nic': [list(x) for x in m['nic']]}
    if r['status'] == 'placed':
        res = scenarios.extract_result(top)
        o.update(res)
        o['nidx'] = list(r['nidx'])
        o['gpu_index'] = [next(i for i, g in enumerate(node.gpus) if g.device_id == d) for d in res['gpus']]
    return o


def reference_queries(scn, ref):
    """{str(k): [outcome of pod i alone on the state after pods 0..k-1]} for the states of query_states."""
    from oracle import ref_loader
    from tests import scenarios
    ref.node.Node.MIN_BUSY_SECS = float(scn.get('min_busy_secs', 30.0))
    nodes = scenarios.build_nodes(scn, ref.node)
    _preuse(scn, nodes)
    names = list(nodes)
    matcher = ref.matcher.Matcher()
    out, done = {}, 0
    for k in query_states(scn):
        for pod, now in zip(scn['pods'][done:k], scn['now'][done:k]):          # the stream up to the state
            top = scenarios.build_top(pod, ref.cfg)
            with contextlib.redirect_stdout(io.StringIO()):
                ref_loader.attempt_scheduling(ref, matcher, nodes, top, pod['groups'], now)
        done = k
        row = []
        # the nodes' locks and loggers are shared by the copies (they cannot be copied), everything else is copied
        lock_type = type(threading.Lock())
        shared = {id(v): v for n in nodes.values() for v in vars(n).values() if isinstance(v, (logging.Logger, lock_type))}
        for pod, now in zip(scn['pods'], scn['now']):                           # every pod alone on that state
            alone = copy.deepcopy(nodes, dict(shared))
            top = scenarios.build_top(pod, ref.cfg)
            with contextlib.redirect_stdout(io.StringIO()):
                r = ref_loader.attempt_scheduling(ref, ref.matcher.Matcher(), alone, top, pod['groups'], now)
            row.append(_outcome(names, alone, r, top))
        out[str(k)] = row
    ref.node.Node.MIN_BUSY_SECS = 30.0
    return out


def make_query():
    from oracle import ref_loader
    ref = ref_loader.load()
    doc = {name: [reference_queries(s, ref) for s in scns] for name, scns in query_streams()}
    seen = {}
    for rows in doc.values():
        for per in rows:
            for outs in per.values():
                for o in outs:
                    seen[o['status']] = seen.get(o['status'], 0) + 1
    print('outcomes', seen)
    live._save('query', doc)


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    make_query()
