"""The oracle of ``nhd_plan_scenarios_releases`` and an oracle stand-in that answers it.  TEST INFRASTRUCTURE.

``oracle_scenario_releases`` plans one ``solver.Scenario`` with ``releases`` as ``plan_oracle.oracle_scenario`` plans
a scenario, with ``plan_oracle.oracle_releases``' counter rules.  ``DeparturesPlanner`` is ``plan_oracle.OraclePlanner``
with scenarios that carry releases answered by it, so that ``NHDScheduler.ForecastDepartures`` runs in the
``-m "not gpu"`` suite.  Never used by the product."""
import numpy as np

from nhd_b200 import wire
from nhd_b200.solver import Scenario
from oracle import binding
from tests import explain_oracle
from tests.plan_oracle import OraclePlanner, _nic_bits, grown, mapped, oracle_scenario


def oracle_scenario_releases(recs, speed, sc, base=0, busy=30.0, explain=False):
    """One scenario with ``releases`` (``(tracked, pods_used, releases)``, ``Scenario.releases``; None: no tracking) as
    ``oracle_scenario`` plans it, every pod solved alone with ``oracle_releases``' counter rules: each placement on a
    tracked node raises the counters of its claimed NICs, each release of round k (in array order, before round k when
    a pod is still unplaced) gives back its cores, GPUs and hugepages, lowers the counters by its pairings and stamps
    the node busy at its clock; every tracked NIC's bit = counter > 0.  Returns ``(bindings, pod_round, counts or None,
    touched)`` as ``oracle_scenario``, ``counts`` taken at the start of each pod's last attempt."""
    sc = Scenario(*sc)
    pods, now = np.asarray(sc.pods), np.asarray(sc.now, dtype='<f8')
    tracked, pods_used, rels = ((), np.zeros((0, wire.MAX_NICS)), None) if sc.releases is None else sc.releases
    rels = np.zeros(0, dtype=wire.RELEASE_DTYPE) if rels is None else np.asarray(rels, dtype=wire.RELEASE_DTYPE)
    g, ids = grown(recs, sc.edits, sc.adds, base)
    where = np.flatnonzero(ids < len(recs))                            # grown position of each source node
    ex = np.unique(where[np.asarray(list(sc.exclude), dtype=np.int64)])
    n = len(pods)
    lift = n if sc.lift is None else sc.lift
    rounds = [] if sc.rounds is None else [float(c) for c in sc.rounds]
    used = np.asarray(pods_used, dtype=np.int64).reshape(len(tracked), wire.MAX_NICS)
    count = {int(where[t]): used[k].copy() for k, t in enumerate(tracked)}
    out = np.zeros(n, dtype=wire.BINDING_DTYPE)
    counts = np.zeros((n, wire.WHY_COUNT), dtype='<u4')
    touched = set()
    r = g.copy()

    def attempt(i, c):
        nonlocal r
        if explain:
            _, why = explain_oracle.batch(r, speed, pods[[i]], np.array([c]), min_busy_secs=busy)
            counts[i] = explain_oracle.counts(why, 1)[0]
        b, r = binding.solve(r, speed, pods[i:i + 1], np.array([c]), min_busy_secs=busy)
        r = r.copy()
        out[i] = b[0]
        node = int(b[0]['node'])
        if node >= 0:
            touched.add(node)
        if b[0]['status'] == wire.PLACED and node in count:
            for j in range(int(b[0]['n_claimed'])):
                count[node][int(b[0]['claimed_nics'][j])] += 1
            r['nic_inuse'][node] = _nic_bits(count[node], int(r['n_nics'][node]))

    def hold(on):
        nonlocal r
        r = r.copy()
        r['flags'][ex] = (g['flags'][ex] | wire.NODE_MAINTENANCE) if on else g['flags'][ex]

    hold(lift > 0)
    for k in range(n):
        if k == lift:
            hold(False)
        attempt(k, now[k])
    pod_round = np.where(out['status'] == wire.PLACED, 0, len(rounds)).astype('<i4')
    hold(lift == n)
    for k, c in enumerate(rounds, 1):
        idx = np.flatnonzero(out['status'] != wire.PLACED)
        if not len(idx):
            continue
        for rl in rels[rels['round'] == k]:
            node = int(where[int(rl['node'])])
            r = r.copy()
            r['used'][node] &= ~rl['cores']
            r['gpu_used'][node] &= ~rl['gpus']
            if rl['hugepages_gb'] > 0:
                r['free_hugepages_gb'][node] += rl['hugepages_gb']
            count[node] -= rl['nic_pairings'].astype(np.int64)
            r['nic_inuse'][node] = _nic_bits(count[node], int(r['n_nics'][node]))
            r['busy_time'][node] = rl['clock']
            touched.add(node)
        for i in idx:
            attempt(i, c)
        pod_round[idx[out['status'][idx] == wire.PLACED]] = k
    counts[out['status'] != wire.NO_CANDIDATE] = 0
    return mapped(out, ids), pod_round, (counts if explain else None), touched


class DeparturesPlanner(OraclePlanner):
    """``OraclePlanner`` whose ``plan_scenarios`` plans a scenario with ``releases`` with ``oracle_scenario_releases``.
    TEST INFRASTRUCTURE."""

    def plan_scenarios(self, scenarios, source='mirror', explain=False):
        scenarios = [Scenario(*sc) for sc in scenarios]
        rounds = any(sc.rounds is not None for sc in scenarios)
        out, base = [], 0
        for sc in scenarios:
            oracle = oracle_scenario if sc.releases is None else oracle_scenario_releases
            b, rnd, counts, _ = oracle(self._source(source), self._speed, sc, base, self._min_busy, explain=explain)
            out.append((0, -1, b) + ((counts,) if explain else ()) + ((rnd,) if rounds else ()))
            base += 0 if sc.adds is None else len(sc.adds[0])
        return out
