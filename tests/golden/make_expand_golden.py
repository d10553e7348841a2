"""Freeze the UNMODIFIED reference's answer to "if these nodes were added, where would the pending pods go?" into
tests/golden/live/expand.json.gz.

The sessions are those of make_defrag_golden.py (``defrag_sessions``): its ``fragmented_script`` sessions leave GPU pods
pending that one more empty GPU node places.  Each session is played to its end state in the reference, then, per
case, the candidate nodes are inserted into the reference scheduler's node dict at their positions (an ``add_nodes``
step that ``_AddNodes`` teaches tests/sched_harness.py's reference driver while installed; each node built as
``BuildInitialNodeList`` builds one, ``candidate_node``) and one pending scan runs.  The cases of a session
(``expand_cases``):
    one empty copy of each node shape of the session (at most three) at the end, at the front and in the middle;
    1, 2 and 3 copies of the first shape at the end;
    a GPU-less node at the front (it takes CPU-only pods first);
    a four-NUMA GPU node at the end;
    a copy in maintenance, and a copy whose labels do not parse, at the front (both stay unused);
    a copy whose node-group set is the groups the pending pods request, which no node has.
The file records, per case, where each pod the scan attempts (in the scan's order, read from this repository's
scheduler replaying the session with the oracle stand-in) ended, or None, and the reference's own reasons for every
node of the grown dict for the pods that found none (make_plan_reasons_golden.py's ``_Attempts``).  A case in which a
Kubernetes write fails during the scan is left out: make_defrag_golden.py says why.  So is a case in which the reference
itself raises (its ``SetPhysicalIdsFromMapping`` on some NIC mappings, which this repository reports as
``REF_WOULD_CRASH``): there is no reference outcome to compare with.
``NHDScheduler.PlanExpansion`` answers all of one session's cases in one call.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_expand_golden.py
"""
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_defrag_golden import _WriteFailures, defrag_sessions, pending_keys   # noqa: E402
from tests.golden.make_plan_golden import mirror_session   # noqa: E402


def expand_sessions():
    """``defrag_sessions()``: ``(name, script)``."""
    return defrag_sessions()


def _shape_key(spec):
    """A node's shape: its labels apart from the NIC labels' MAC addresses and name-derived values."""
    labels = {k: v for k, v in spec['labels'].items() if 'nfd-extras-nic' not in k}
    nics = sorted('.'.join(k.split('.')[-6:]) for k in spec['labels'] if 'nfd-extras-nic' in k)
    return json.dumps([sorted(labels.items()), nics, spec['hp_alloc']])


def _copy(spec, name, **kw):
    out = copy.deepcopy(spec)
    out.update(name=name, hp_free=spec['hp_alloc'], active=True, **kw)
    return out


def expand_cases(script, names, requested):
    """The cases of one session: ``[{'label', 'nodes': [{'node': tests.scenarios node, 'before': name or None}]}]``.
    ``names``: the session's nodes in order; ``requested``: the node-group names the pending pods request."""
    from tests import scenarios as S
    shapes, seen = [], set()
    for spec in script['nodes']:
        key = _shape_key(spec)
        if key not in seen and spec['hp_alloc'] > 0 and spec.get('active', True) and 'DATA_PLANE_VLAN' in spec['labels']:
            seen.add(key)
            shapes.append(spec)
    shapes = shapes[:3]
    first, middle = names[0], names[len(names) // 2]
    cases = []
    for k, spec in enumerate(shapes):
        for where, before in (('end', None), ('front', first), ('middle', middle)):
            cases.append({'label': f'shape{k}-{where}', 'nodes': [{'node': _copy(spec, f'new{k}'), 'before': before}]})
    for c in (1, 2, 3):
        cases.append({'label': f'copies{c}', 'nodes': [{'node': _copy(shapes[0], f'copy{i}'), 'before': None}
                                                       for i in range(c)]})
    cpu = S.make_node('newcpu', 2, 32, False, 1, (), [('eth0', 100000, 0, 0x10), ('eth1', 100000, 1, 0x20)],
                      hp_alloc=64)
    cases.append({'label': 'gpuless-front', 'nodes': [{'node': cpu, 'before': first}]})
    gpus = [(d, d // 2, 0x10 * (d // 2 + 1)) for d in range(8)]
    nics = [(f'eth{k}', 100000, k, 0x10 * (k + 1)) for k in range(4)]
    four = S.make_node('newnuma4', 4, 32, True, 1, gpus, nics, hp_alloc=64)
    cases.append({'label': 'numa4-end', 'nodes': [{'node': four, 'before': None}]})
    maint = _copy(shapes[0], 'newmaint')
    maint['labels']['sigproc.viasat.io/maintenance'] = 'draining'
    cases.append({'label': 'maintenance-front', 'nodes': [{'node': maint, 'before': first}]})
    broken = _copy(shapes[0], 'newbroken')
    del broken['labels']['DATA_PLANE_VLAN']
    cases.append({'label': 'labels-front', 'nodes': [{'node': broken, 'before': first}]})
    grouped = _copy(shapes[0], 'newgroups')
    grouped['labels']['NHD_GROUP'] = '.'.join(requested or ['default'])
    cases.append({'label': 'groups-middle', 'nodes': [{'node': grouped, 'before': middle}]})
    return cases


def candidate_node(node_cls, spec):
    """A node the scheduler does not hold yet, built from a ``tests.scenarios`` node as ``BuildInitialNodeList`` builds
    one (NHDScheduler.py:74-98): ``Node(name, active)``, ``ParseLabels``, ``SetHugepages``; labels that do not parse,
    no hugepages or an exception leave it inactive."""
    v = node_cls(spec['name'], spec.get('active', True))
    try:
        if not v.ParseLabels(spec['labels']):
            v.active = False
        elif spec['hp_alloc'] == 0 or not v.SetHugepages(spec['hp_alloc'], spec['hp_free']):
            v.active = False
    except Exception:
        v.active = False
    return v


def add_nodes(sched, node_cls, nodes):
    """``nodes`` (``[{'node': tests.scenarios node, 'before': name or None}]``) built by ``candidate_node`` and inserted
    into ``sched.nodes`` right before the node named ``before`` (None: at the end), nodes with the same ``before`` in
    list order.  The dict is changed in place: the placement loop walks it in this order."""
    items = list(sched.nodes.items())
    for d in nodes:
        names = [n for n, _ in items]
        items.insert(len(items) if d['before'] is None else names.index(d['before']),
                     (d['node']['name'], candidate_node(node_cls, d['node'])))
    sched.nodes.clear()
    sched.nodes.update(items)


class _AddNodes:
    """While installed, the reference driver of tests/sched_harness.py (``run_reference``) plays the step
    ``{'op': 'add_nodes', 'nodes': [...]}`` as ``add_nodes`` on the reference scheduler it is running, with the
    reference's own ``Node`` class.  The driver's other steps are untouched."""

    def __enter__(self):
        from oracle import ref_sched_loader
        from tests import sched_harness as H
        self.loader, self.feed, self.rpc = ref_sched_loader, H._RefFeed, H._RefFeed._Rpc
        self.make, self.get, self.rpc_get = ref_sched_loader.make_scheduler, H._RefFeed.get, H._RefFeed._Rpc.get
        made, make, get, rpc_get = [], self.make, self.get, self.rpc_get

        def making(*args, **kw):
            made.append(make(*args, **kw))
            return made[-1]

        def play(feed):                                   # the scheduler reads the two queues in turn: either may meet it
            while feed.i < len(feed.steps) and feed.steps[feed.i]['op'] == 'add_nodes':
                add_nodes(made[-1], feed.ref.node.Node, feed.steps[feed.i]['nodes'])
                feed.i += 1

        def getting(feed, *args, **kw):
            play(feed)
            return get(feed, *args, **kw)

        def rpc_getting(rpc, *args, **kw):
            play(rpc.f)
            return rpc_get(rpc, *args, **kw)
        self.loader.make_scheduler, self.feed.get, self.rpc.get = making, getting, rpc_getting
        return self

    def __exit__(self, *exc):
        self.loader.make_scheduler, self.feed.get, self.rpc.get = self.make, self.get, self.rpc_get


def grown_names(names, nodes):
    """The node order with the candidate nodes inserted (``add_nodes``' rule)."""
    out = list(names)
    for d in nodes:
        out.insert(len(out) if d['before'] is None else out.index(d['before']), d['node']['name'])
    return out


def candidates(sched, cases, node_cls):
    """Per golden case, the ``PlanExpansion`` scenario (``[(node, before)]``, nodes built with ``node_cls``) and the
    grown node order."""
    names = list(sched.nodes)
    return [([(candidate_node(node_cls, d['node']), d['before']) for d in c['nodes']], grown_names(names, c['nodes']))
            for c in cases]


def expand_session(item):
    from tests import helpers
    from tests import sched_harness as H
    from tests.golden.make_plan_reasons_golden import _Attempts, _last, _run
    name, script = item
    sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
    try:
        names = list(sched.nodes)
        pending = pending_keys(sched)
        requested = sorted({g for ns, pod in pending for g in k8s.GetPodNodeGroups(pod, ns)} - {'default'})
    finally:
        sched.close()
    cases = expand_cases(script, names, requested)
    out, left_out, crashed, helped = [], 0, 0, 0
    with _Attempts() as att, _WriteFailures() as failures, _AddNodes():
        start = len(_run(att, script))
        prefix_failures = failures.n
        for case in cases:
            failures.n = 0
            steps = script['steps'] + [{'op': 'add_nodes', 'nodes': case['nodes']}, {'op': 'idle'}]
            att.log = []
            try:
                doc = H.run_reference(dict(script, steps=steps))
            except TypeError:                   # the reference's own crash in SetPhysicalIdsFromMapping (Node.py:833)
                crashed += 1
                continue
            log = list(att.log)
            if failures.n != prefix_failures:
                left_out += 1
                continue
            assert list(doc['nodes']) == grown_names(names, case['nodes']), (name, case['label'])
            where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
            placed = [where.get(f'{ns}/{pod}') for ns, pod in pending]
            added = {d['node']['name'] for d in case['nodes']}
            helped += any(p in added for p in placed)
            out.append(dict(case, placed=placed, reasons=_last(log, start, set(pending))))
    print(name, len(pending), 'pending,', len(out), 'cases kept,', left_out, 'left out,', crashed, 'crashed,', helped,
          'placing on an added node', flush=True)
    return {'name': name, 'pending': [list(p) for p in pending], 'cases': out}, len(out), left_out, helped


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        res = pool.map(expand_session, expand_sessions(), chunksize=1)
    cases, left_out, helped = (sum(r[i] for r in res) for i in (1, 2, 3))
    print(cases, 'cases,', left_out, 'left out for a failed Kubernetes write,', helped, 'placing a pod on an added node')
    assert helped >= 20, helped
    live._save('expand', {'sessions': [r[0] for r in res]})


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    main()
