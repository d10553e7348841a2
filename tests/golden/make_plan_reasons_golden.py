"""Freeze the UNMODIFIED reference's own reasons for dropping nodes, for the pods its drains and defrag workflows leave
without a node, into tests/golden/live/plan_reasons.json.gz.

The sessions and the appended steps are those of make_drains_golden.py (one node drained, its pods re-created) and
make_defrag_golden.py (drained, re-created, back in service, one pending scan after each delay).  Every reference
``AttemptScheduling`` is recorded with a ``logging.Handler`` on the reference Matcher's logger, and every node given
the code of the record that dropped it, as make_explain_golden.py does (its ``DROPS``, and the ``InitialNodeFilter``
restatement for the group and active stages, taken when the attempt starts).  An attempt that reached ``FindNode`` and
in which every node is dropped is one in which ``FindNode`` found no node; an attempt that ended before it (a pod or
config that cannot be read) has no reasons.  The run of the session alone makes as many attempts as the
prefix of every appended run (the reference is deterministic), so what follows them belongs to the appended steps:
    a re-created pod    its first attempt after the prefix;
    a pending pod       its last attempt (the scan after the node's return).
The file holds, per case, {"ns/name": one digit per node} for the pods whose attempt dropped every node: ``moved``
for the re-created pods, ``pending`` (defrag) for the scanned ones.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_plan_reasons_golden.py
"""
import logging
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_defrag_golden import (PER_SESSION, SHORT_DELAY, _WriteFailures, defrag_sessions,  # noqa: E402
                                             pending_keys, return_steps)
from tests.golden.make_explain_golden import DROPS, _Records      # noqa: E402
from tests.golden.make_plan_golden import drain_nodes, drain_sessions, drain_steps, mirror_session   # noqa: E402


class _Attempts:
    """Records every reference ``AttemptScheduling`` while installed: ``[(ns, name, codes or None)]``, codes being one
    digit per node when every node was dropped."""

    def __enter__(self):
        from oracle import ref_sched_loader
        ref = ref_sched_loader.load()
        self.log = []
        self.handler = _Records()
        self.logger = logging.getLogger(ref.matcher.__name__)
        self.logger.addHandler(self.handler)
        self.logger.setLevel(logging.DEBUG)
        logging.disable(logging.NOTSET)
        self.cls = ref.sched.NHDScheduler
        self.orig = self.cls.AttemptScheduling
        outer = self

        def attempt(sched, podname, ns):
            groups = set(sched.k8s.GetPodNodeGroups(podname, ns))
            codes = {}
            for n, v in sched.nodes.items():                   # InitialNodeFilter, NHDScheduler.py:240-241
                if not set(v.groups) & groups:
                    codes[n] = 0
                elif not v.active:
                    codes[n] = 1
            outer.handler.msgs = []
            reached, find = [], sched.matcher.FindNode

            def found(*args, **kw):                              # the attempt got as far as FindNode
                reached.append(True)
                return find(*args, **kw)
            sched.matcher.FindNode = found
            try:
                ok = outer.orig(sched, podname, ns)
            finally:
                del sched.matcher.FindNode
            if not reached:
                codes = {}
            for msg in outer.handler.msgs:
                for rx, code in DROPS:
                    m = rx.match(msg)
                    if m and m.group(1) not in codes:
                        codes[m.group(1)] = code
            full = not ok and sched.nodes and sorted(codes) == sorted(sched.nodes)
            outer.log.append((ns, podname, ''.join(str(codes[n]) for n in sched.nodes) if full else None))
            return ok
        self.cls.AttemptScheduling = attempt
        return self

    def __exit__(self, *exc):
        self.cls.AttemptScheduling = self.orig
        self.logger.removeHandler(self.handler)
        logging.disable(logging.CRITICAL)


def _run(att, script):
    from tests import sched_harness as H
    att.log = []
    H.run_reference(script)
    return list(att.log)


def _first_after(log, start, pods):
    out = {}
    for ns, name, codes in log[start:]:
        if (ns, name) in pods and (ns, name) not in out:
            out[(ns, name)] = codes
    return {f'{ns}/{name}': c for (ns, name), c in out.items() if c is not None}


def _last(log, start, pods):
    out = {}
    for ns, name, codes in log[start:]:
        if (ns, name) in pods:
            out[(ns, name)] = codes
    return {f'{ns}/{name}': c for (ns, name), c in out.items() if c is not None}


def drains_session(item):
    from tests import helpers
    name, script, _ = item
    sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
    try:
        nodes = drain_nodes(sched, k8s, PER_SESSION)
        plans = [(n,) + drain_steps(script, sched, [n]) for n in nodes]
    finally:
        sched.close()
    with _Attempts() as att:
        start = len(_run(att, script))
        drains = [{'node': node, 'moved': _first_after(_run(att, dict(script, steps=script['steps'] + steps)), start,
                                                       set(pods))}
                  for node, steps, pods in plans]
    print(name, sum(len(d['moved']) for d in drains), 'pods without a node', flush=True)
    return {'name': name, 'drains': drains}


def defrag_session(item):
    from tests import helpers
    name, script = item
    sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
    try:
        nodes = drain_nodes(sched, k8s, PER_SESSION)
        drains = [(n,) + drain_steps(script, sched, [n]) for n in nodes]
        pending = set(pending_keys(sched))
    finally:
        sched.close()
    delays = []
    with _Attempts() as att, _WriteFailures() as failures:
        start = len(_run(att, script))
        prefix_failures = failures.n
        for delay in (float(script['min_busy_secs']), SHORT_DELAY):
            out = []
            for node, steps, moved in drains:
                failures.n = 0
                log = _run(att, dict(script, steps=script['steps'] + steps + return_steps(node, delay)))
                if failures.n != prefix_failures:              # left out of defrag.json.gz too
                    continue
                out.append({'node': node, 'moved': _first_after(log, start, set(moved)),
                            'pending': _last(log, start, pending)})
            delays.append({'delay': delay, 'drains': out})
    print(name, sum(len(c['moved']) + len(c['pending']) for d in delays for c in d['drains']), 'pods without a node',
          flush=True)
    return {'name': name, 'delays': delays}


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        drains = pool.map(drains_session, drain_sessions(), chunksize=1)
        defrag = pool.map(defrag_session, defrag_sessions(), chunksize=1)
    live._save('plan_reasons', {'drains': drains, 'defrag': defrag})


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    main()
