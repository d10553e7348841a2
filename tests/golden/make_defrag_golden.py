"""Freeze the UNMODIFIED reference's answer to "if this node were drained and put back in service, where would its pods
go, and would the pending pods then place?" into tests/golden/live/defrag.json.gz.

The sessions are those of make_plan_golden.py (``drain_sessions``), played to the same end state, plus seeded sessions
in which GPU pods are left pending by fragmentation (``fragmented_script``).  For each of up to eight nodes
holding the most pods (``drain_nodes``' rule), and at two delays (the session's ``min_busy_secs``, the first moment the
released node takes GPU pods again, and 5 s, inside its busy window), one reference run of the session followed by the
maintenance workflow on that node alone:
    NODE_MAINT_START, the node's pods deleted and re-created (``drain_steps``), NODE_MAINT_END, the clock moved on by
    the delay, one pending scan.
The file records where each re-created pod and each pod the scan attempts (in the scan's order, read from this
repository's scheduler replaying the session with the oracle stand-in) ended, or None.  A case in which a Kubernetes
write fails during the appended steps (an injected ``nad`` / ``gpumap`` / ``annotate`` / ``bind`` failure of a pending
pod) is left out: the reference then releases what the pod took on its node, which a plan does not model.  Read
failures are kept: a pod whose object or config cannot be read fails the same way in a plan.
``NHDScheduler.PlanDefrag`` answers all of one session's cases at one delay in one call, before any drain.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_defrag_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_plan_golden import DRAIN_DT, drain_nodes, drain_sessions, drain_steps, mirror_session   # noqa: E402

PER_SESSION = 8
SHORT_DELAY = 5.0


def fragmented_script(seed):
    """A session in which GPU pods are left pending by fragmentation: four GPU nodes (two or four GPUs per NUMA node)
    filled first-fit with one-GPU pods (one at a time, the clock moving past each busy window), then all but one pod per
    NUMA node deleted, the clock moved past the busy windows, then pods that need every GPU of one NUMA node.  Every
    node then holds free GPUs, none a free NUMA node's worth; draining one node moves its two pods into the other
    nodes' gaps and frees it.  No injected Kubernetes failures."""
    from tests import scenarios as S
    rng = np.random.default_rng(seed)
    per_numa = int(rng.choice([2, 4]))
    nodes = []
    for i in range(4):
        gpus = [(d, d // per_numa, 0x10 * (d // per_numa + 1)) for d in range(2 * per_numa)]
        nics = [(f'eth{k}', 100000, k, 0x10 * (k + 1)) for k in range(2)]
        nodes.append(S.make_node(f'n{i}', 2, 32, bool(rng.random() < 0.5), 1, gpus, nics, hp_alloc=64, hp_free=64))
    if rng.random() < 0.5:                                # a CPU-only node first: the GPU-less pass goes there first
        nodes.insert(0, S.make_node('cpu0', 2, 32, False, 1, (), [('eth0', 100000, 0, 0x10)], hp_alloc=64, hp_free=64))
    counter = [0]

    def pod(n_gpus):
        counter[0] += 1
        spec = S.make_pod([S.make_group([], int(rng.integers(1, 3)), [int(rng.integers(0, 2))] * n_gpus, 0)],
                          int(rng.integers(0, 2)), False, 'NUMA', int(rng.choice([0, 2])))
        return {'op': 'add_pod', 'ns': 'ns0', 'name': f'pod{counter[0]}', 'uid': f'u{counter[0]}', 'fail': [],
                'pod': spec}
    small = [pod(1) for _ in range(4 * 2 * per_numa)]
    steps = []
    for p in small:                                       # one at a time, past each other's busy window: first-fit
        steps += [p, {'op': 'idle'}, {'op': 'clock', 'dt': 31.0}]
    for i in range(4):                                    # every node keeps one pod on each NUMA node
        keep = {int(rng.integers(0, per_numa)), per_numa + int(rng.integers(0, per_numa))}
        for k in range(2 * per_numa):
            if k not in keep:
                victim = small[i * 2 * per_numa + k]['name']
                steps += [{'op': 'watch', 'type': 'NHD_WATCH_TYPE_TRIAD_POD_DELETE',
                           'pod': {'ns': 'ns0', 'name': victim, 'uid': 'gone'}},
                          {'op': 'delete_pod', 'ns': 'ns0', 'name': victim}]
    steps.append({'op': 'clock', 'dt': 100.0})
    steps += [pod(per_numa) for _ in range(int(rng.integers(1, 3)))] + [pod(1) for _ in range(int(rng.integers(0, 2)))]
    steps += [{'op': 'idle'}, {'op': 'clock', 'dt': DRAIN_DT}]
    return {'nodes': nodes, 'min_busy_secs': float(rng.choice([30.0, 0.0])), 'clock0': 1000.0, 'init': [],
            'steps': steps, 'codec': 'json'}


def defrag_sessions():
    """``drain_sessions()`` and the ``fragmented_script`` sessions, each as ``(name, script)``."""
    out = [(name, script) for name, script, _ in drain_sessions()]
    return out + [(f'json{seed}_fragmented', fragmented_script(seed)) for seed in (41, 42, 43, 44, 45, 46)]


def pending_keys(sched):
    """The pods the next pending scan attempts, in its order: ``[(ns, name)]``."""
    phase = sched._service_pods()
    wanted = sched._wanted(phase)
    return [(k[0], k[1]) for k in phase if wanted(k)]


def return_steps(node, delay):
    return [{'op': 'watch', 'type': 'NHD_WATCH_TYPE_NODE_MAINT_END', 'node': node},
            {'op': 'clock', 'dt': delay}, {'op': 'idle'}]


class _WriteFailures:
    """Counts the Kubernetes writes of the fake manager that fail, across every manager made while it is installed."""

    def __enter__(self):
        from tests import fake_k8s
        self.n = 0
        self._cls = fake_k8s.FakeK8s
        self._write, self._bind = self._cls._write, self._cls.BindPodToNode
        outer = self

        def write(k8s, *args):
            ok = outer._write(k8s, *args)
            outer.n += not ok
            return ok

        def bind(k8s, *args):
            ok = outer._bind(k8s, *args)
            outer.n += not ok
            return ok
        self._cls._write, self._cls.BindPodToNode = write, bind
        return self

    def __exit__(self, *exc):
        self._cls._write, self._cls.BindPodToNode = self._write, self._bind


def defrag_session(item):
    """The cases of one session: ``(session document, cases, cases left out, cases in which a pending pod places that
    does not place without the defrag)``."""
    from tests import helpers, sched_harness as H
    name, script = item
    sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
    try:
        nodes = drain_nodes(sched, k8s, PER_SESSION)
        drains = [(n,) + drain_steps(script, sched, [n]) for n in nodes]
        pending = pending_keys(sched)
    finally:
        sched.close()
    cases = left_out = helped = 0
    with _WriteFailures() as failures:
        H.run_reference(script)
        prefix_failures = failures.n
        # where the re-created pods went while the node was in maintenance (the scan may move a pod that found no node
        # there onto the node once it is back)
        moved_to = {}
        for node, steps, moved in drains:
            doc = H.run_reference(dict(script, steps=script['steps'] + steps))
            where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
            moved_to[node] = [where.get(f'{ns}/{pod}') for ns, pod in moved]
            assert node not in moved_to[node], (name, node)
        delays = []
        for delay in (float(script['min_busy_secs']), SHORT_DELAY):
            alone = H.run_reference(dict(script, steps=script['steps'] + return_steps(nodes[0], delay)[1:])) \
                if nodes else None
            before = {p for st in alone['nodes'].values() for p in st['pods']} if alone else set()
            out = []
            for node, steps, moved in drains:
                failures.n = 0
                doc = H.run_reference(dict(script, steps=script['steps'] + steps + return_steps(node, delay)))
                if failures.n != prefix_failures:
                    left_out += 1
                    continue
                where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
                pending_to = [where.get(f'{ns}/{pod}') for ns, pod in pending]
                cases += 1
                if all(m is not None for m in moved_to[node]):
                    helped += any(p is not None and f'{ns}/{pod}' not in before
                                  for (ns, pod), p in zip(pending, pending_to))
                out.append({'node': node, 'moved': [list(p) for p in moved], 'moved_to': moved_to[node],
                            'pending_to': pending_to})
            delays.append({'delay': delay, 'drains': out})
    print(name, len(nodes), 'nodes,', len(pending), 'pending,', cases, 'cases kept,', helped, 'helped', flush=True)
    return {'name': name, 'pending': [list(p) for p in pending], 'delays': delays}, cases, left_out, helped


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        res = pool.map(defrag_session, defrag_sessions(), chunksize=1)
    cases, left_out, helped = (sum(r[i] for r in res) for i in (1, 2, 3))
    print(cases, 'cases,', left_out, 'left out for a failed Kubernetes write,', helped,
          'in which a pending pod places that does not place without the defrag')
    assert helped >= 10, helped
    live._save('defrag', {'sessions': [r[0] for r in res]})


if __name__ == '__main__':
    main()
