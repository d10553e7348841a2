"""Freeze the UNMODIFIED reference's answer to "where do the pods of this one node go if it alone is drained?" into
tests/golden/live/drains.json.gz.

The sessions are those of make_plan_golden.py (``drain_sessions``), played to the same end state.  There, up to the
eight nodes holding the most pods (``drain_nodes``' rule) are each drained on their own: for every such node, one
reference run of the session followed by the drain of that node alone (``drain_steps``), recording per re-created pod
the node the reference bound it to or None.  ``NHDScheduler.PlanDrains`` answers all of them in one call before any
drain.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_drains_golden.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_plan_golden import drain_nodes, drain_sessions, drain_steps, mirror_session   # noqa: E402

PER_SESSION = 8


def main():
    from tests import helpers, sched_harness as H
    sessions = []
    for name, script, _ in drain_sessions():
        sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
        try:
            nodes = drain_nodes(sched, k8s, PER_SESSION)
            plans = [(n,) + drain_steps(script, sched, [n]) for n in nodes]
        finally:
            sched.close()
        drains = []
        for node, steps, pods in plans:
            doc = H.run_reference(dict(script, steps=script['steps'] + steps))
            where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
            outcome = [where.get(f'{ns}/{pod}') for ns, pod in pods]
            assert node not in outcome, (name, node)
            drains.append({'node': node, 'pods': [list(p) for p in pods], 'outcome': outcome})
        sessions.append({'name': name, 'drains': drains})
        print(name, len(drains), 'nodes,', sum(len(d['pods']) for d in drains), 'pods,',
              sum(o is None for d in drains for o in d['outcome']), 'without a node,',
              sum(all(o is not None for o in d['outcome']) for d in drains), 'drainable')
    live._save('drains', {'sessions': sessions})


if __name__ == '__main__':
    main()
