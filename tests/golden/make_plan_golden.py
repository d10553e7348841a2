"""Freeze the UNMODIFIED reference's answer to "where do the pods of these nodes go if the nodes are drained?" into
tests/golden/live/plan.json.gz.

Each session is a seeded ``sched_harness.random_script`` of one flavour (mixed, wild, vf, big, and libconfig text)
played to its end, then one more pending scan and a 5-second clock step, so that nodes that just took a pod are inside
their busy window.  Then the drain: the nodes holding the most pods (``drain_nodes``) get ``NODE_MAINT_START``; every
pod on them (nodes in that order, pods in ``Node.pod_info`` order) is deleted (the delete event, which releases it
while its annotations can still be read, then the Kubernetes object) and re-created with the same request and a create
event, one after the other at that clock.  The reference's ``run()`` schedules each re-created pod as it arrives; the
file records, per re-created pod, the node the reference bound it to or None.  The pods' order is read from this repository's scheduler replaying the same
session with the oracle stand-in (``mirror_session``); tests/test_scheduler.py pins that replay to the reference.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_plan_golden.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402

DRAIN_DT = 5.0


def drain_sessions():
    """(name, prefix script, number of nodes to drain), shared with tests/test_plan.py."""
    from tests import sched_harness as H
    out = []
    for flavor, codec, seeds in (('mixed', 'json', (21, 22, 23, 24)), ('wild', 'json', (25, 26, 27, 28)),
                                 ('vf', 'json', (29, 30, 31)), ('big', 'json', (32, 33, 34)),
                                 ('mixed', 'triad', (35,)), ('wild', 'triad', (36,))):
        for seed in seeds:
            script = H.random_script(seed, flavor, codec=codec)
            # the session up to its closing RPCs, a last pending scan, and the clock the drain happens at
            script['steps'] = script['steps'][:-4] + [{'op': 'idle'}, {'op': 'clock', 'dt': DRAIN_DT}]
            out.append((f'{codec}{seed}_{flavor}', script, 2 + seed % 2))
    return out


def mirror_session(script, solver_factory):
    """This repository's scheduler after ``script`` (as ``sched_harness.run_mirror`` plays it), left open with its
    fake Kubernetes manager and clock: ``(sched, k8s, clock)``.  The caller closes ``sched``."""
    import nhd_b200.CfgTopology as cfg_mod
    import nhd_b200.Node as node_mod
    from nhd_b200.NHDScheduler import NHDScheduler
    from tests import fake_k8s, sched_harness as H
    node_mod.Node.MIN_BUSY_SECS = float(script['min_busy_secs'])
    clock = H.Clock(script['clock0'])
    k8s = fake_k8s.FakeK8s(script['nodes'], codec=script.get('codec', 'json'))
    for st in script['init']:
        H.apply_k8s_op(k8s, clock, st)
    if script.get('codec', 'json') == 'triad':
        from nhd_b200.TriadCfgParser import TriadCfgParser
        parser = lambda cfgtype, cfgstr: TriadCfgParser(cfgstr, False)          # noqa: E731
    else:
        parser = lambda cfgtype, cfgstr: fake_k8s.JsonCfgParser(cfgstr, cfg_mod)  # noqa: E731

    def make():
        s = NHDScheduler(k8s, parser, solver_factory=solver_factory, clock=clock)
        s.Startup()
        return s
    s = make()
    for st in script['steps']:
        op = st['op']
        if op in H.K8S_OPS:
            H.apply_k8s_op(k8s, clock, st)
        elif op == 'watch':
            s.HandleWatchItem({k: v for k, v in st.items() if k != 'op'})
        elif op == 'rpc':
            s.ParseRPCReq(st['msg'], H.RpcSink())
        elif op == 'idle':
            s.CheckPendingPods()
        elif op == 'restart':
            s.close()
            s = make()
    return s, k8s, clock


def drain_nodes(sched, k8s, n):
    """The ``n`` nodes holding the most pods (ties in node order) whose pods all still have a Kubernetes object."""
    cands = [name for name, v in sched.nodes.items()
             if v.pod_info and all((ns, pod) in k8s.pods for (pod, ns) in v.pod_info)]
    cands.sort(key=lambda name: -len(sched.nodes[name].pod_info))
    return cands[:n]


def drain_steps(script, sched, nodes):
    """The drain of ``nodes`` as script steps, and the re-created pods ``[(ns, name)]`` in their order."""
    spec = {}
    for st in script['init'] + script['steps']:
        if st['op'] == 'add_pod':
            spec[(st['ns'], st['name'])] = st['pod']
    pods = [(ns, pod) for n in nodes for (pod, ns) in sched.nodes[n].pod_info]
    steps = [{'op': 'watch', 'type': 'NHD_WATCH_TYPE_NODE_MAINT_START', 'node': n} for n in nodes]
    for ns, name in pods:
        steps += [{'op': 'watch', 'type': 'NHD_WATCH_TYPE_TRIAD_POD_DELETE', 'pod': {'ns': ns, 'name': name, 'uid': 'gone'}},
                  {'op': 'delete_pod', 'ns': ns, 'name': name}]
    for ns, name in pods:
        uid = f'r-{ns}-{name}'
        steps += [{'op': 'add_pod', 'ns': ns, 'name': name, 'uid': uid, 'fail': [], 'pod': spec[(ns, name)]},
                  {'op': 'watch', 'type': 'NHD_WATCH_TYPE_TRIAD_POD_CREATE', 'pod': {'ns': ns, 'name': name, 'uid': uid}}]
    return steps, pods


def main():
    from tests import helpers, sched_harness as H
    sessions = []
    for name, script, n in drain_sessions():
        sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
        try:
            nodes = drain_nodes(sched, k8s, n)
            steps, pods = drain_steps(script, sched, nodes)
        finally:
            sched.close()
        doc = H.run_reference(dict(script, steps=script['steps'] + steps))
        where = {p: node for node, st in doc['nodes'].items() for p in st['pods']}
        outcome = [where.get(f'{ns}/{pod}') for ns, pod in pods]
        assert not any(o in nodes for o in outcome), name
        sessions.append({'name': name, 'drain': nodes, 'pods': [list(p) for p in pods], 'outcome': outcome})
        print(name, nodes, len(pods), 'pods,', sum(o is None for o in outcome), 'without a node')
    live._save('plan', {'sessions': sessions})


if __name__ == '__main__':
    main()
