"""The oracles of the what-if calls, and the oracle stand-in that answers them.  TEST INFRASTRUCTURE.

``oracle_alone`` (a batch of one per pod), ``oracle_scenario`` (one ``solver.Scenario``: edits, additions, exclusions
lifted at a pod, later rounds) and ``oracle_releases`` (one solve per pod with the signed NIC counters) compute, with
the C oracle, what the GPU calls must return byte for byte.  ``OraclePlanner`` puts them behind ``Solver``'s interface
so that the scheduler's previews, plans and forecasts run in the ``-m "not gpu"`` suite.  Never used by the product."""
import numpy as np

from nhd_b200 import wire
from nhd_b200.solver import Scenario
from oracle import binding
from tests import explain_oracle, helpers


def excluded(recs, exclude):
    """A copy of ``recs`` with the nodes ``exclude`` in maintenance (the reference's NODE_MAINT_START)."""
    out = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE).copy()
    idx = np.asarray(list(exclude), dtype=np.int64)
    out['flags'][idx] |= wire.NODE_MAINTENANCE
    return out


def grown(recs, edits=None, adds=None, base=0):
    """The grown scratch records of a scenario: ``recs`` with the edits applied and the added records inserted, each
    right before source node ``at`` (added nodes at one position in array order).  Returns ``(records, ids)``, ``ids``
    the index each grown node reports: its source index, or ``len(recs) + base + k`` for the scenario's k-th
    addition (``base``: the additions of the call before this scenario)."""
    r = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE).copy()
    if edits is not None and len(edits[0]):
        r[np.asarray(edits[0], dtype=np.int64)] = edits[1]
    at, arecs = (np.zeros(0, dtype=np.int64), r[:0]) if adds is None else adds
    at = np.asarray(at, dtype=np.int64)
    assert (np.diff(at) >= 0).all()
    n = len(r)
    ids = np.arange(n, dtype=np.int64)
    if len(at):
        ids = np.insert(ids, at, n + base + np.arange(len(at)))    # each in front of source node at[k]
    out = np.zeros(len(ids), dtype=wire.NODE_DTYPE)
    src = ids < n
    out[src] = r
    out[~src] = np.asarray(arecs, dtype=wire.NODE_DTYPE)[ids[~src] - n - base]
    return out, ids


def mapped(b, ids):
    b = b.copy()
    on = b['node'] >= 0
    b['node'][on] = ids[b['node'][on]]
    return b


def oracle_alone(recs, speed, pods, now, busy=30.0, threads=1):
    """Pod i solved alone on a fresh copy of ``recs``, for every i."""
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    for i in range(len(pods)):
        out[i] = binding.solve(recs, speed, pods[i:i + 1], now[i:i + 1], min_busy_secs=busy, threads=threads)[0][0]
    return out


def oracle_scenario(recs, speed, sc, base=0, busy=30.0, threads=1, explain=False):
    """One scenario (a ``Scenario`` or a tuple of its fields) with the C oracle: the five steps on the grown copy of
    ``recs`` (edits applied, additions inserted, the excluded nodes in maintenance for the pods before the lift and
    back after), then per round clock the pods not placed yet solved again in order (exclusions held at the last pod
    held again).  ``base``: the additions of the call before this scenario.  Returns ``(bindings, pod_round, counts or
    None, touched)``, node indices mapped back; ``counts`` with ``explain``: per pod the explanation oracle's per-reason
    node counts at its last attempt (whose bindings must be the solve's, byte for byte); ``touched`` the grown nodes any
    attempt chose."""
    sc = Scenario(*sc)
    pods, now = np.asarray(sc.pods), np.asarray(sc.now, dtype='<f8')
    g, ids = grown(recs, sc.edits, sc.adds, base)
    where = np.flatnonzero(ids < len(recs))                            # grown position of each source node
    ex = np.unique(where[np.asarray(list(sc.exclude), dtype=np.int64)])
    n = len(pods)
    lift = n if sc.lift is None else sc.lift
    rounds = [] if sc.rounds is None else [float(c) for c in sc.rounds]
    kw = dict(min_busy_secs=busy, threads=threads)
    out = np.zeros(n, dtype=wire.BINDING_DTYPE)
    counts = np.zeros((n, wire.WHY_COUNT), dtype='<u4')
    touched = set()

    def phase(r, idx, clocks):
        b, after = binding.solve(r, speed, pods[idx], clocks, **kw)
        if explain:
            eb, why = explain_oracle.batch(r, speed, pods[idx], clocks, **kw)
            assert eb.tobytes() == b.tobytes(), helpers.first_binding_diff(eb, b)
            counts[idx] = explain_oracle.counts(why, len(idx))
        out[idx] = b
        touched.update(int(x) for x in b['node'] if x >= 0)
        return after
    r = g.copy()
    flags = r['flags'][ex].copy()
    r = excluded(r, ex)
    if lift:
        r = phase(r, np.arange(lift), now[:lift])
    r['flags'][ex] = flags
    if lift < n:
        r = phase(r, np.arange(lift, n), now[lift:])
    pod_round = np.where(out['status'] == wire.PLACED, 0, len(rounds)).astype('<i4')
    for k, c in enumerate(rounds, 1):
        idx = np.flatnonzero(out['status'] != wire.PLACED)
        if not len(idx):
            continue
        held = r['flags'][ex].copy()
        if lift == n:
            r = excluded(r, ex)
        r = phase(r, idx, np.full(len(idx), c))
        r['flags'][ex] = held
        pod_round[idx[out['status'][idx] == wire.PLACED]] = k
    return mapped(out, ids), pod_round, (counts if explain else None), touched


def _nic_bits(count, n_nics):
    return int(sum(1 << i for i in range(n_nics) if count[i] > 0))


def oracle_releases(recs, speed, pods, now, rounds, tracked, pods_used, releases, exclude=(), busy=30.0, explain=False,
                    solve_one=None):
    """``(bindings, pod_round, counts or None, cuts)``: every pod solved alone on the records the pods before it left,
    the counters of the tracked nodes raised by each placement's claimed NICs and lowered by each release's pairings,
    each tracked NIC's bit = counter > 0.  ``cuts[r]``: the placements of round r that claimed a NIC whose counter was
    <= -1 (where the batch path cuts).  ``solve_one(records, pod, clock)`` -> ``(binding, records)``; the C oracle by
    default."""
    if solve_one is None:
        def solve_one(r, pod, clock):
            b, r = binding.solve(r, speed, pod[None], np.array([clock]), min_busy_secs=busy)
            return b[0], r
    r = excluded(recs, exclude)
    count = {int(n): np.asarray(pods_used[t], dtype=np.int64).copy() for t, n in enumerate(tracked)}
    n = len(pods)
    out = np.zeros(n, dtype=wire.BINDING_DTYPE)
    counts = np.zeros((n, wire.WHY_COUNT), dtype='<u4')
    cuts = [0] * (len(rounds) + 1)

    def attempt(k, idx, clocks, last):
        nonlocal r
        for i, c in zip(idx, clocks):
            if explain and last:
                _, why = explain_oracle.batch(r, speed, pods[[i]], np.array([c]), min_busy_secs=busy)
                counts[i] = explain_oracle.counts(why, 1)[0]
            b, r = solve_one(r, pods[i], c)
            out[i] = b
            node = int(b['node'])
            if b['status'] == wire.PLACED and node in count:
                for j in range(int(b['n_claimed'])):
                    nic = int(b['claimed_nics'][j])
                    cuts[k] += int(count[node][nic] <= -1)
                    count[node][nic] += 1
                r = r.copy()
                r['nic_inuse'][node] = _nic_bits(count[node], int(r['n_nics'][node]))

    def release(rl):
        nonlocal r
        r = r.copy()
        node = int(rl['node'])
        r['used'][node] &= ~rl['cores']
        r['gpu_used'][node] &= ~rl['gpus']
        if rl['hugepages_gb'] > 0:
            r['free_hugepages_gb'][node] += rl['hugepages_gb']
        count[node] -= rl['nic_pairings'].astype(np.int64)
        r['nic_inuse'][node] = _nic_bits(count[node], int(r['n_nics'][node]))
        r['busy_time'][node] = rl['clock']

    attempt(0, range(n), now, not len(rounds))
    pod_round = np.where(out['status'] == wire.PLACED, 0, len(rounds)).astype('<i4')
    for k, c in enumerate(rounds, 1):
        idx = np.flatnonzero(out['status'] != wire.PLACED)
        if not len(idx):
            break
        for rl in releases[releases['round'] == k]:
            release(rl)
        attempt(k, idx, np.full(len(idx), c), k == len(rounds))
        pod_round[idx[out['status'][idx] == wire.PLACED]] = k
    counts[out['status'] != wire.NO_CANDIDATE] = 0
    return out, pod_round, (counts if explain else None), cuts


class OraclePlanner(helpers.OracleSolver):
    """The oracle stand-in with every what-if call ``Solver`` has but ``plan_batch_rounds`` (the scheduler then takes
    the scenario call): queries, plans, explanations, scenarios of any fields and releases, each on a copy of the
    records (``source='snapshot'``: of the last snapshot).  TEST INFRASTRUCTURE."""

    def _source(self, source):
        return self._snap if source == 'snapshot' else self._recs

    def query_batch(self, pods, now, source='mirror'):
        return oracle_alone(self._source(source), self._speed, np.asarray(pods), np.asarray(now, dtype='<f8'),
                            self._min_busy)

    def solve_batch(self, pods, now):
        self._last = (np.asarray(pods).copy(), np.asarray(now, dtype='<f8').copy())
        return super().solve_batch(pods, now)

    def explain_batch(self):
        return oracle_scenario(self._snap, self._speed, ((),) + self._last, busy=self._min_busy, explain=True)[2]

    def plan_batch(self, pods, now, source='mirror', exclude=(), explain=False):
        out, _, counts, _ = oracle_scenario(self._source(source), self._speed, (exclude, pods, now), busy=self._min_busy,
                                            explain=True)
        return (out, counts) if explain else out

    def plan_scenarios(self, scenarios, source='mirror', explain=False):
        scenarios = [Scenario(*sc) for sc in scenarios]
        rounds = any(sc.rounds is not None for sc in scenarios)
        out, base = [], 0
        for sc in scenarios:
            b, rnd, counts, _ = oracle_scenario(self._source(source), self._speed, sc, base, self._min_busy,
                                                explain=explain)
            out.append((0, -1, b) + ((counts,) if explain else ()) + ((rnd,) if rounds else ()))
            base += 0 if sc.adds is None else len(sc.adds[0])
        return out

    def plan_batch_releases(self, pods, now, round_clocks, tracked, pods_used, releases, source='mirror', exclude=(),
                            explain=False):
        b, rnd, counts, _ = oracle_releases(self._source(source), self._speed, np.asarray(pods),
                                            np.asarray(now, dtype='<f8'), [float(c) for c in round_clocks],
                                            list(tracked), np.asarray(pods_used).reshape(len(tracked), wire.MAX_NICS),
                                            np.asarray(releases, dtype=wire.RELEASE_DTYPE), [int(i) for i in exclude],
                                            self._min_busy, explain)
        return (b, rnd, counts) if explain else (b, rnd)
