"""``Matcher.FindNode`` under the reference scheduler's calling pattern (one call per pod on the filtered node dict,
``NHDScheduler.py:235-247,277-304``) with the change counters of ``nhd_b200/tracking.py``: only the nodes that
changed since the previous call are packed and uploaded, and every answer equals that of a matcher that packs the
whole dict on every call.  Runs on the GPU (``-m gpu``) and, in the CPU suite, on the emulated device."""
import numpy as np
import pytest

import nhd_b200.CfgTopology as cfg_mod
import nhd_b200.Node as node_mod
from tests import scenarios


def _initial_filter(nodes, groups):
    """NHDScheduler.InitialNodeFilter (NHDScheduler.py:235-247): active nodes sharing a group with the pod, in order."""
    return {k: v for k, v in nodes.items() if v.active and set(v.groups) & set(groups)}


def _plain(match):
    if match == (None,):
        return match
    return match[0], {k: v for k, v in match[1].items() if k != '_nhd_binding'}


def _session(nmod, cmod, seed, n_nodes, n_steps, flavor):
    from nhd_b200.Matcher import Matcher
    rng = np.random.default_rng(seed)
    scn = scenarios.random_scenario(seed, n_nodes=n_nodes, n_pods=n_steps, flavor=flavor)
    nmod.Node.MIN_BUSY_SECS = 0.0
    inc, full = Matcher(track=True), Matcher(track=False)
    try:
        nodes = scenarios.build_nodes(scn, nmod)
        names = list(nodes)
        placed = []
        now = 1000.0
        calls = found = 0
        seen = set()
        for step, pod in enumerate(scn['pods']):
            now += 1.0
            act = rng.integers(0, 10)
            if act == 0 and placed:                                    # a pod goes away (NHDScheduler.py:107-135)
                node, top = placed.pop(int(rng.integers(0, len(placed))))
                node.AddResourcesFromTopology(top)
            elif act == 1:                                             # cordon / uncordon (NHDScheduler.py:541-549)
                n = nodes[names[int(rng.integers(0, len(names)))]]
                n.active = not n.active
            elif act == 2:                                             # maintenance label (NHDScheduler.py:557-564)
                n = nodes[names[int(rng.integers(0, len(names)))]]
                n.maintenance = not n.maintenance
            elif act == 3:                                             # node group label changed (NHDScheduler.py:570)
                nodes[names[int(rng.integers(0, len(names)))]].SetGroups('default.' + ('a', 'b')[int(rng.integers(0, 2))])
            nl = _initial_filter(nodes, pod['groups'])
            if not nl:
                continue
            top = scenarios.build_top(pod, cmod)
            packed_before = inc.stats['packed']
            a = inc.FindNode(nl, top, now=now)
            b = full.FindNode(nl, top, now=now)
            calls += 1
            assert _plain(a) == _plain(b), (step, _plain(a), _plain(b))
            fresh = len(set(nl) - seen)                               # nodes the matcher has never been shown
            seen.update(nl)
            assert inc.stats['packed'] - packed_before <= fresh + 4, (step, fresh, inc.stats)   # not the whole dict again
            if a == (None,):
                continue
            found += 1
            if rng.integers(0, 5) == 0:
                continue                                               # the caller gives up before applying anything
            node = nodes[a[0]]
            node.busy_time = now                                       # SetBusy (NHDScheduler.py:289)
            try:
                nic_list = node.SetPhysicalIdsFromMapping(a[1], top)   # (:292)
            except IndexError:
                continue
            if nic_list is None:
                continue
            node.ClaimPodNICResources(list({x[0] for x in nic_list}))  # (:302-304)
            placed.append((node, top))
        assert calls >= n_steps // 2 and found >= calls // 3, (calls, found)
        assert full.stats['packed'] >= calls * 2 and inc.stats['packed'] < full.stats['packed'] // 3, (inc.stats, full.stats)
        assert inc.stats['full_loads'] <= 8, inc.stats            # the device order settles after a few distinct filter results
    finally:
        nmod.Node.MIN_BUSY_SECS = 30.0
        for m in (inc, full):
            if m._solver is not None:
                m._solver.close()


@pytest.mark.gpu
@pytest.mark.parametrize('flavor', ['mixed', 'wild'])
def test_incremental_matcher_equals_full_repack_on_mirror_nodes(flavor):
    _session(node_mod, cfg_mod, 9100 + len(flavor), n_nodes=24, n_steps=70, flavor=flavor)
