"""A pod beyond the tuple limit that depends on the cluster (numa^(groups+1) tuples, include/nhd_b200.h): the library
refuses the whole call and names the pod.  Every ``NHDScheduler`` entry point drops that pod and goes on with the rest:
the batch fails it loudly, previews and plans map it to None and leave the pod unmarked.

The cluster has a 4-NUMA node, ``quad``, and four 2-NUMA nodes.  A 4-group pod only passes the limit while ``quad`` is
out of service, so ``four`` is deployed during a maintenance window of ``quad``; afterwards every call that counts
``quad`` refuses it.  ``-m gpu``: the CUDA library (on the CPU, the emulated device of
``tests/test_emulated_device.py``)."""
import pytest

from tests import fake_k8s, scenarios, sched_harness as H

pytestmark = pytest.mark.gpu

NICS = [(f'eth{k}', 100000, k, 0x10 * (k + 1)) for k in range(4)]
SMALL = scenarios.make_pod([scenarios.make_group(pairs=((10, 10),), workers=1)], misc=1)
FOUR = scenarios.make_pod([scenarios.make_group(pairs=((5, 5),), workers=1) for _ in range(4)], misc=1)
HUGE = scenarios.make_pod([scenarios.make_group(workers=40)], misc=1)          # no NUMA node has 40 free cores
PENDING = [('p0', SMALL), ('p1', FOUR), ('p2', SMALL), ('p3', HUGE), ('p4', FOUR), ('p5', SMALL)]
KEYS = [('a', name, f'u{name}') for name, _ in PENDING]
REFUSED = {('a', 'p1'), ('a', 'p4')}
KEPT = [k for k in KEYS if (k[0], k[1]) not in REFUSED]


def _session():
    """The scheduler after the deployment, ``quad`` back in service, the pods of ``PENDING`` waiting; and the node that
    holds ``four``."""
    from nhd_b200.NHDScheduler import NHDScheduler
    import nhd_b200.CfgTopology as cfg_mod
    nodes = [scenarios.make_node('quad', 4, 64, True, 1, nics=NICS)] + \
        [scenarios.make_node(f'n{i}', 2, 32, True, 2, nics=NICS[:2]) for i in (1, 2, 3, 4)]
    k8s = fake_k8s.FakeK8s(nodes)
    s = NHDScheduler(k8s, lambda t, c: fake_k8s.JsonCfgParser(c, cfg_mod), clock=H.Clock(1000.0))
    s.BuildInitialNodeList()
    s.HandleWatchItem({'type': 'NHD_WATCH_TYPE_NODE_MAINT_START', 'node': 'quad'})
    k8s.add_pod('a', 'four', FOUR, uid='ufour')
    for i in range(5):
        k8s.add_pod('a', f'd{i}', SMALL, uid=f'ud{i}')
    s.CheckPendingPods()
    s.HandleWatchItem({'type': 'NHD_WATCH_TYPE_NODE_MAINT_END', 'node': 'quad'})
    bound = {b[1]: b[2] for b in k8s.binds}
    assert len(bound) == 6 and not s.unsupported_pods, (bound, s.unsupported_pods)
    holder = bound['four']
    assert len(s.nodes[holder].pod_info) > 1               # ``four`` shares its node with a small pod
    for name, pod in PENDING:
        k8s.add_pod('a', name, pod, uid=f'u{name}')
    return s, k8s, holder


def _unmarked(s):
    assert not s.unsupported_pods and s.failed_schedule_count == 0


def _without_refused(d):
    return {k: v for k, v in d.items() if k not in REFUSED}


def test_preview_maps_a_refused_pod_to_none():
    s, _, _ = _session()
    try:
        got = s.PreviewPods(KEYS)
        assert list(got) == [(k[0], k[1]) for k in KEYS]
        assert all(got[k] is None for k in REFUSED)
        assert _without_refused(got) == s.PreviewPods(KEPT)
        assert got[('a', 'p0')] is not None and got[('a', 'p3')] is None
        _unmarked(s)
    finally:
        s.close()


def test_plan_pods_maps_a_refused_pod_to_none():
    s, _, _ = _session()
    try:
        placement, reasons = s.PlanPods(KEYS)
        assert all(placement[k] is None for k in REFUSED) and not REFUSED & set(reasons)
        want = s.PlanPods(KEPT)
        assert (_without_refused(placement), reasons) == want
        assert placement[('a', 'p0')] is not None and ('a', 'p3') in reasons
        _unmarked(s)
    finally:
        s.close()


def test_plan_drain_maps_a_refused_pod_to_none():
    s, _, holder = _session()
    try:
        placement, reasons = s.PlanDrain([holder])
        assert list(placement) == [(ns, pod) for (pod, ns) in s.nodes[holder].pod_info]
        assert placement.pop(('a', 'four')) is None and ('a', 'four') not in reasons
        assert placement and all(v is not None and v != holder for v in placement.values())
        _unmarked(s)
    finally:
        s.close()


def test_plan_drains_falls_back_to_the_single_plan_for_a_refused_group():
    """The scenario call counts every node and refuses each group that moves ``four``.  The single plan counts the nodes
    outside the group: with ``quad`` in the group it places ``four``, without it ``four`` maps to None."""
    s, _, holder = _session()
    try:
        other = next(n for n, v in s.nodes.items() if v.pod_info and n != holder)
        groups = [(holder,), (holder, 'quad'), (other,)]
        got = s.PlanDrains(groups)
        assert got == {g: s.PlanDrain(list(g))[0] for g in groups}
        assert got[(holder,)][('a', 'four')] is None and got[(holder, 'quad')][('a', 'four')] is not None
        _unmarked(s)
    finally:
        s.close()


def test_plan_defrag_maps_refused_pods_to_none():
    """``four`` among the moved pods: it maps to None, the group's other pods go where ``PlanDrain`` sends them, and the
    pending pods are not planned.  ``p1`` and ``p4`` in the pending tail: they map to None and the rest is the plan
    without them."""
    s, _, holder = _session()
    try:
        other = next(n for n, v in s.nodes.items() if v.pod_info and n != holder)
        groups = [(holder,), (other,)]
        got = s.PlanDefrag(KEYS, groups)
        moved, pending = got[(holder,)]
        assert moved[('a', 'four')] is None and moved == s.PlanDrain([holder])[0] and pending is None
        moved, pending = got[(other,)]
        assert all(v is not None for v in moved.values()) and pending is not None
        assert all(pending[k] is None for k in REFUSED)
        assert (moved, _without_refused(pending)) == s.PlanDefrag(KEPT, [(other,)])[(other,)]
        _unmarked(s)
    finally:
        s.close()


def test_schedule_batch_fails_a_refused_pod_and_schedules_the_rest():
    s, k8s, _ = _session()
    try:
        s.CheckPendingPods()
        assert [b[1] for b in k8s.binds[6:]] == ['p0', 'p2', 'p5']
        assert [p[1] for p in s.unsupported_pods] == ['p1', 'p4'] and s.failed_schedule_count == 3
        assert all('tuple' in p[2] for p in s.unsupported_pods)
    finally:
        s.close()
