"""The oracle of ``nhd_plan_scenarios_arrivals`` and an oracle stand-in that answers it.  TEST INFRASTRUCTURE.

``oracle_scenario_arrivals`` plans one ``solver.Scenario`` with ``arrive`` as
``departures_oracle.oracle_scenario_releases`` plans a scenario, with each later pod first attempted alone at its own
clock, in its gap, by clock among that gap's releases.  ``ArrivalsPlanner`` is ``DeparturesPlanner`` with scenarios
that carry arrivals answered by it, so that ``NHDScheduler.ForecastArrivals`` runs in the ``-m "not gpu"`` suite.
Never used by the product."""
import numpy as np

from nhd_b200 import wire
from nhd_b200.solver import Scenario
from oracle import binding
from tests import explain_oracle
from tests.departures_oracle import DeparturesPlanner
from tests.plan_oracle import _nic_bits, grown, mapped


def oracle_scenario_arrivals(recs, speed, sc, base=0, busy=30.0, explain=False):
    """One scenario with ``arrive`` (None: every pod pending at the start) and ``releases`` (None: no tracking), every
    pod solved alone with ``oracle_releases``' counter rules.  Round 0 solves the round-0 pods at their clocks, the
    exclusions held for the pods before ``lift``.  Gap g then plays, merged by clock, its releases (in array order) and
    the first attempt of each pod arriving in it at its own clock, a release first at an equal clock; each release only
    while a pod is unplaced or not yet attempted.  Scan g retries at its clock every attempted pod not placed, in pod
    order.  After round 0 the exclusions stay held exactly when ``lift`` is the pod count.  Returns ``(bindings,
    pod_round, counts or None, pod_clock)``: the round whose arrival or scan placed each pod (else the round count),
    ``counts`` taken at the start of each pod's last attempt, ``pod_clock`` that attempt's clock (the placing one)."""
    sc = Scenario(*sc)
    pods, now = np.asarray(sc.pods), np.asarray(sc.now, dtype='<f8')
    n = len(pods)
    arrive = np.zeros(n, dtype=np.int64) if sc.arrive is None else np.asarray(sc.arrive, dtype=np.int64)
    tracked, pods_used, rels = ((), np.zeros((0, wire.MAX_NICS)), None) if sc.releases is None else sc.releases
    rels = np.zeros(0, dtype=wire.RELEASE_DTYPE) if rels is None else np.asarray(rels, dtype=wire.RELEASE_DTYPE)
    g, ids = grown(recs, sc.edits, sc.adds, base)
    where = np.flatnonzero(ids < len(recs))
    ex = np.unique(where[np.asarray(list(sc.exclude), dtype=np.int64)])
    lift = n if sc.lift is None else sc.lift
    rounds = [] if sc.rounds is None else [float(c) for c in sc.rounds]
    used = np.asarray(pods_used, dtype=np.int64).reshape(len(tracked), wire.MAX_NICS)
    count = {int(where[t]): used[k].copy() for k, t in enumerate(tracked)}
    out = np.zeros(n, dtype=wire.BINDING_DTYPE)
    counts = np.zeros((n, wire.WHY_COUNT), dtype='<u4')
    clock = np.zeros(n, dtype='<f8')
    tried = np.zeros(n, dtype=bool)
    pod_round = np.full(n, len(rounds), dtype='<i4')
    r = g.copy()

    def attempt(i, c, k):
        nonlocal r
        if explain:
            _, why = explain_oracle.batch(r, speed, pods[[i]], np.array([c]), min_busy_secs=busy)
            counts[i] = explain_oracle.counts(why, 1)[0]
        b, r = binding.solve(r, speed, pods[i:i + 1], np.array([c]), min_busy_secs=busy)
        r = r.copy()
        out[i], clock[i], tried[i] = b[0], c, True
        node = int(b[0]['node'])
        if b[0]['status'] == wire.PLACED:
            pod_round[i] = k
            if node in count:
                for j in range(int(b[0]['n_claimed'])):
                    count[node][int(b[0]['claimed_nics'][j])] += 1
                r['nic_inuse'][node] = _nic_bits(count[node], int(r['n_nics'][node]))

    def hold(on):
        nonlocal r
        r = r.copy()
        r['flags'][ex] = (g['flags'][ex] | wire.NODE_MAINTENANCE) if on else g['flags'][ex]

    def release(rl):
        nonlocal r
        if ((out['status'] == wire.PLACED) & tried).all():
            return
        node = int(where[int(rl['node'])])
        r = r.copy()
        r['used'][node] &= ~rl['cores']
        r['gpu_used'][node] &= ~rl['gpus']
        if rl['hugepages_gb'] > 0:
            r['free_hugepages_gb'][node] += rl['hugepages_gb']
        count[node] -= rl['nic_pairings'].astype(np.int64)
        r['nic_inuse'][node] = _nic_bits(count[node], int(r['n_nics'][node]))
        r['busy_time'][node] = rl['clock']

    hold(lift > 0)
    for k in np.flatnonzero(arrive == 0):
        if k == lift:
            hold(False)
        attempt(k, now[k], 0)
    hold(lift == n)
    for k, c in enumerate(rounds, 1):
        todo = list(rels[rels['round'] == k])
        for i in np.flatnonzero(arrive == k):
            while todo and todo[0]['clock'] <= now[i]:
                release(todo.pop(0))
            attempt(i, now[i], k)
        for rl in todo:
            release(rl)
        for i in np.flatnonzero((arrive <= k) & (out['status'] != wire.PLACED)):
            attempt(i, c, k)
    counts[out['status'] != wire.NO_CANDIDATE] = 0
    return mapped(out, ids), pod_round, (counts if explain else None), clock


class ArrivalsPlanner(DeparturesPlanner):
    """``DeparturesPlanner`` whose ``plan_scenarios`` plans every scenario with ``oracle_scenario_arrivals`` when any
    scenario has ``arrive``, each result then ending with the pod rounds and the pod clocks.  TEST INFRASTRUCTURE."""

    def plan_scenarios(self, scenarios, source='mirror', explain=False):
        scenarios = [Scenario(*sc) for sc in scenarios]
        if all(sc.arrive is None for sc in scenarios):
            return super().plan_scenarios(scenarios, source, explain)
        out, base = [], 0
        for sc in scenarios:
            b, rnd, counts, clock = oracle_scenario_arrivals(self._source(source), self._speed, sc, base,
                                                             self._min_busy, explain=explain)
            out.append((0, -1, b) + ((counts,) if explain else ()) + (rnd, clock))
            base += 0 if sc.adds is None else len(sc.adds[0])
        return out
