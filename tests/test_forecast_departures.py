"""Forecasts under several departure schedules side by side (``nhd_plan_scenarios_releases``,
``Solver.plan_scenarios`` with ``Scenario.releases``, ``NHDScheduler.ForecastDepartures``).

The contract is ``nhd_plan_scenarios_rounds`` with each scenario's deployed pods ending between its rounds, on its own
records and signed NIC pod counters: byte for byte each pod's last attempt, the round that placed it, and the reasons
of the pods whose last attempt found no node.  ``oracle_scenario_releases`` (tests/departures_oracle.py) is that plan:
one oracle solve per pod, ``ClaimPodNICResources`` on the counters after each placement, ``AddResourcesFromTopology``
+ ``SetBusy`` for each release.  The chain of evidence:
  * on the CPU emulation of the device (tests/emu), both lane orders, seeded calls that mix scenarios with edits,
    additions, exclusions held or lifted, rounds, releases, negative counters and none, with and without reasons, equal
    that oracle; with no track and release offsets the call is ``nhd_plan_scenarios_rounds``; one plain scenario is
    ``nhd_plan_batch_releases``, also where that call cuts; every malformed argument is refused and nothing of the
    handle moves;
  * ``ForecastDepartures`` equals ``ForecastPending`` where the two overlap, on the oracle stand-in and on the device;
  * on the GPU the same cases, and config 4 at full size after its solve (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import _lib, wire
from nhd_b200.solver import Scenario
from tests import helpers
from tests.departures_oracle import DeparturesPlanner, oracle_scenario_releases
from tests.plan_oracle import oracle_scenario
from tests.test_forecast_releases import release_cases, release_of
from tests.test_plan import _emu_lib
from tests.test_query import _filter_words, _gpu_cases, emu_cases, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def test_the_symbol_is_declared_and_exported():
    from nhd_b200 import build
    build.build()
    text = open(os.path.join(ROOT, 'include', 'nhd_b200.h')).read()
    assert 'int32_t nhd_plan_scenarios_releases(nhd_handle* h, int32_t source, int32_t n_scenarios' in text
    assert 'nhd_plan_scenarios_releases' in _lib.EXPORTS and hasattr(_lib.load(), 'nhd_plan_scenarios_releases')


# ---------------------------------------------------------------------------------------------- the cases
def departure_calls(recs, speed, pods, now, busy, seed):
    """``(state, [Scenario])`` calls on one stream, from ``release_cases``: per release case one call of seven
    scenarios on its state, each a random run of the pending pods: the case's releases alone, with an exclusion held
    to the end or lifted at a pod, with an edited node (its fresh record), with an added node (a copy of a fresh
    record), tracking without releases, and no releases at all."""
    rng = np.random.default_rng(1000 + seed)
    out = []
    for st, tail, clock, rounds, tracked, used, rels in release_cases(recs, speed, pods, now, busy, seed):
        if not len(tail):
            continue
        n = len(st)
        rel_nodes = {int(x) for x in rels['node']}
        free = [k for k in range(n) if k not in rel_nodes and k not in tracked]

        def pick():
            k = int(rng.integers(1, min(len(tail), 10) + 1))
            idx = np.sort(rng.choice(len(tail), k, replace=False))
            return tail[idx], clock[idx]
        full = (tracked, used, rels)
        scs = [Scenario((), tail, clock, None, None, None, rounds, full)]
        p, c = pick()
        scs.append(Scenario([int(rng.integers(n))], p, c, None, None, None, rounds, full))
        p, c = pick()
        scs.append(Scenario([int(rng.integers(n))], p, c, int(rng.integers(len(p) + 1)), None, None, rounds, full))
        if free:
            e = int(rng.choice(free))
            p, c = pick()
            scs.append(Scenario((), p, c, None, ([e], recs[[e]]), None, rounds, full))
        p, c = pick()
        k = int(rng.integers(n))
        scs.append(Scenario((), p, c, None, None, ([int(rng.integers(n + 1))], recs[[k]]), rounds, full))
        p, c = pick()
        scs.append(Scenario((), p, c, None, None, None, rounds, (tracked, used, rels[:0])))
        p, c = pick()
        scs.append(Scenario((), p, c, None, None, None, rounds, None))
        out.append((st, scs))
    return out


def oracle_call(st, speed, scs, busy, explain):
    """Per scenario ``(bindings, pod_round, counts)`` of the oracle, added nodes numbered across the call."""
    res, base = [], 0
    for sc in scs:
        oracle = oracle_scenario if sc.releases is None else oracle_scenario_releases
        b, rnd, counts, _ = oracle(st, speed, sc, base, busy, explain=explain)
        res.append((b, rnd, counts))
        base += 0 if sc.adds is None else len(sc.adds[0])
    return res


def check_calls(s, calls, speed, busy, where=''):
    """Every call equals the oracle on every scenario, with reasons and without.  Returns (pods compared, pods placed
    at a round >= 1 in a scenario with releases)."""
    n = later = 0
    for j, (st, scs) in enumerate(calls):
        s.load_nodes(st)
        got = s.plan_scenarios(scs, explain=True)
        plain = s.plan_scenarios(scs)
        want = oracle_call(st, speed, scs, busy, True)
        for k, ((code, pod, b, rows, rnd), (wb, wrnd, wrows), sc, pl) in enumerate(zip(got, want, scs, plain)):
            assert code == 0, (where, j, k, code, pod)
            assert b.tobytes() == wb.tobytes(), (where, j, k, helpers.first_binding_diff(wb, b))
            assert (rnd == wrnd).all(), (where, j, k, rnd, wrnd)
            assert (rows == wrows).all(), (where, j, k, np.flatnonzero((rows != wrows).any(1)))
            assert pl[2].tobytes() == b.tobytes() and (pl[3] == rnd).all(), (where, j, k)
            n += len(b)
            if sc.releases is not None and len(sc.releases[2]):
                later += int(((b['status'] == wire.PLACED) & (rnd >= 1)).sum())
    return n, later


class _ViaReleases:
    """A library whose ``nhd_plan_scenarios_rounds`` is ``nhd_plan_scenarios_releases`` with NULL track and release
    arrays: ``Solver.plan_scenarios`` through it tests the first identity of the header."""
    def __init__(self, L):
        self._L = L

    def __getattr__(self, name):
        return getattr(self._L, name)

    def nhd_plan_scenarios_rounds(self, *a):
        return self._L.nhd_plan_scenarios_releases(*a[:17], None, None, None, None, None, *a[17:])


def check_identities(s, calls, cases, speed, busy):
    """Null track and release offsets: ``nhd_plan_scenarios_rounds`` byte for byte, reasons included.  One scenario
    with no edits, no additions and no lift: ``nhd_plan_batch_releases``' bindings and rounds, byte for byte.  Returns
    the cuts the batch path makes on those cases (the oracle loop's count of claims at a counter <= -1)."""
    from tests.plan_oracle import oracle_releases
    for st, scs in calls:
        s.load_nodes(st)
        plain = [Scenario(*sc[:7]) for sc in scs]
        a = s.plan_scenarios(plain, explain=True)
        L = s._L
        s._L = _ViaReleases(L)
        try:
            b = s.plan_scenarios(plain, explain=True)
        finally:
            s._L = L
        assert all(x[:2] == y[:2] and all(u.tobytes() == v.tobytes() for u, v in zip(x[2:], y[2:])) for x, y in zip(a, b))
    cuts = 0
    for st, p, c, rounds, tracked, used, rels in cases:
        if not len(p):
            continue
        s.load_nodes(st)
        want, wrnd = s.plan_batch_releases(p, c, rounds, tracked, used, rels)
        (code, _, got, grnd), = s.plan_scenarios([Scenario((), p, c, None, None, None, rounds, (tracked, used, rels))])
        assert code == 0 and got.tobytes() == want.tobytes(), helpers.first_binding_diff(want, got)
        assert (grnd == wrnd).all()
        cuts += sum(oracle_releases(st, speed, p, c, rounds, tracked, used, rels, busy=busy)[3])
    return cuts


def check_refusals(s, st, scs, speed, busy):
    """Every malformed argument is NHD_ERR_INVALID and leaves records, snapshot, staged batch, bindings, bitmaps,
    explanations, timing and counters as they were; a plan afterwards equals one on a fresh handle."""
    import ctypes
    from nhd_b200.solver import Solver, SolverError
    sc, other = scs[0], scs[-1]
    tracked, used, rels = sc.releases
    rounds = sc.rounds
    assert len(rels) and len(rounds) >= 1 and other.releases is None
    s.load_nodes(st)
    s.snapshot()
    b = s.solve_batch(sc.pods, sc.now)
    timing, counters = s.timing(), s.debug_counters()

    def state():
        words, pt = _filter_words(s)
        return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                s.explain_batch().tobytes())
    before = state()

    def refused(what, bad, tamper=None):
        L = s._L
        if tamper is not None:
            s._L = _Tamper(L, tamper)
        try:
            with pytest.raises(SolverError) as e:
                s.plan_scenarios([other, bad], source='snapshot')
        finally:
            s._L = L
        assert e.value.code == wire.ERR_INVALID and what in str(e.value), (what, str(e.value))

    def rel(f):
        r = rels.copy()
        f(r)
        return sc._replace(releases=(tracked, used, r))
    last = len(rounds)
    refused('outside [1,', rel(lambda r: r['round'].__setitem__(0, 0)))
    refused('outside [1,', rel(lambda r: r['round'].__setitem__(0, last + 1)))
    refused('not finite', rel(lambda r: r['clock'].__setitem__(0, np.nan)))
    if len(rels) > 1:
        refused('go down', rel(lambda r: r['clock'].__setitem__(1, r['clock'][0] - 1e-3)))
    t0 = float(np.max(sc.now))
    refused('outside the gap', rel(lambda r: (r['round'].__setitem__(0, 1), r['clock'].__setitem__(0, t0 - 1.0))))
    refused('outside the gap', rel(lambda r: (r['round'].__setitem__(0, 1), r['clock'].__setitem__(0, rounds[0] + 1.0))))
    refused('without rounds', sc._replace(rounds=None))
    refused('not tracked', sc._replace(releases=(tracked[1:], used[1:], rels)))
    refused('tracked twice', sc._replace(releases=(tracked + tracked[:1], np.concatenate([used, used[:1]]), rels)))
    refused('outside the', sc._replace(releases=([len(st)] + tracked[1:], used, rels)))
    node = int(rels[0]['node'])
    refused('edits', sc._replace(edits=([node], st[[node]])))
    t = tracked.index(node)
    if st['n_nics'][node]:
        flip = used.copy()
        flip[t, 0] = 0 if st['nic_inuse'][node] & 1 else 1
        refused('disagrees', sc._replace(releases=(tracked, flip, rels)))
    if st['n_nics'][node] < wire.MAX_NICS:
        beyond = used.copy()
        beyond[t, wire.MAX_NICS - 1] = 1
        refused('disagrees', sc._replace(releases=(tracked, beyond, rels)))
    lc = int(st['phys_cores'][node]) * (2 if st['flags'][node] & wire.NODE_SMT else 1)
    if lc < 256:
        refused('beyond node', rel(lambda r: r['cores'][0].__setitem__(lc >> 6, r['cores'][0][lc >> 6] | np.uint64(1) << np.uint64(lc & 63))))
    if int(st['n_gpus'][node]) < 16:
        refused('beyond node', rel(lambda r: r['gpus'].__setitem__(0, r['gpus'][0] | (1 << int(st['n_gpus'][node])))))
    if int(st['n_nics'][node]) < wire.MAX_NICS:
        refused('beyond node', rel(lambda r: r['nic_pairings'][0].__setitem__(int(st['n_nics'][node]), 1)))

    def word(addr, k, v):
        ctypes.cast(addr, ctypes.POINTER(ctypes.c_int32))[k] = v

    def at(k, v):
        def f(a):
            a = list(a)
            a[k] = v
            return a
        return f
    refused('start at 0', sc, lambda a: (word(a[17], 0, 1), a)[1])
    refused('start at 0', sc, lambda a: (word(a[20], 0, 1), a)[1])
    refused('go down', sc, lambda a: (word(a[17], 1, len(tracked) + 1), a)[1])
    refused('go down', sc, lambda a: (word(a[20], 1, len(rels) + 1), a)[1])
    for k in (18, 19, 21):                   # tracked, pods_used, releases NULL with entries
        L = s._L
        s._L = _Tamper(L, at(k, None))
        try:
            with pytest.raises(SolverError) as e:
                s.plan_scenarios([other, sc], source='snapshot')
        finally:
            s._L = L
        assert e.value.code == wire.ERR_INVALID
    assert state() == before
    assert s.timing() == timing and (s.debug_counters() == counters).all()
    # a plan between a solve and its explanations moves nothing either, and equals one on a fresh handle
    got = s.plan_scenarios(scs, source='snapshot', explain=True)
    assert state() == before
    fresh = Solver(speed, min_busy_secs=busy)
    try:
        fresh.load_nodes(st)
        want = fresh.plan_scenarios(scs, explain=True)
    finally:
        fresh.close()
    assert all(x[:2] == y[:2] and all(u.tobytes() == v.tobytes() for u, v in zip(x[2:], y[2:])) for x, y in zip(got, want))
    s.restore()
    s.solve_staged()
    assert s.fetch_bindings().tobytes() == b.tobytes()


class _Tamper:
    """A library whose ``nhd_plan_scenarios_releases`` gets its arguments through ``f`` first (malformed offsets and
    NULL arrays that ``Solver.plan_scenarios`` never sends)."""
    def __init__(self, L, f):
        self._L, self._f = L, f

    def __getattr__(self, name):
        return getattr(self._L, name)

    def nhd_plan_scenarios_releases(self, *a):
        return self._L.nhd_plan_scenarios_releases(*self._f(a))


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
from nhd_b200.solver import Solver
from tests.test_forecast_departures import check_calls, check_identities, check_refusals, departure_calls
from tests.test_forecast_releases import release_cases
from tests.test_query import emu_cases, packed
tot = [0] * 3
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        calls = departure_calls(recs, speed, pods, now, busy, j)
        tot[:2] = [a + b for a, b in zip(tot, check_calls(s, calls, speed, busy, j))]
        if j %% 3 == 0:
            tot[2] += check_identities(s, calls, release_cases(recs, speed, pods, now, busy, j), speed, busy)
        if j == 1:
            check_refusals(s, *calls[3], speed, busy)
    finally:
        s.close()
print('compared', *tot)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_departures_on_the_emulated_device_equal_the_oracle(lane_order):
    """``emu_cases()`` streams, half deployed: calls mixing edits, additions, exclusions held and lifted,
    rounds, releases, negative starting counters, tracking alone and no releases, with reasons and without; both
    identities (one of them where the batch path cuts); the refusals."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=2400)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    n, later, cuts = (int(x) for x in res.stdout.split()[-3:])
    assert n > 300 and later > 10 and cuts > 0, res.stdout


# ---------------------------------------------------------------------------------------------- the scheduler
def _schedules_against_the_reference(factory, limit=None):
    """``ForecastDepartures`` with every departure schedule of a session in one call equals the reference's scans with
    those deletes played between them (tests/golden/live/releases.json.gz), the same with an added node or none per
    schedule (departures.json.gz), and with the candidate nodes of a session and no departures the reference's scans
    on the grown cluster (forecast.json.gz): the scan and node of every pending
    pod and the reasons at the last scan of those no scan placed; nothing is written.  Each result also equals
    ``ForecastPending`` on its own."""
    from tests.golden import make_live_golden
    from tests.golden.make_expand_golden import candidates
    from tests.golden.make_forecast_golden import SCANS as F_SCANS, VARIANTS, forecast_sessions
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import SCANS, release_sessions
    from tests.test_plan_reasons import _counted
    n = 0
    golden = make_live_golden.load('releases')['sessions']
    for (name, script), want in list(zip(release_sessions(), golden))[:limit]:
        keys = [tuple(k) for k in want['pending']]
        for period in sorted({c['period'] for c in want['cases']}):
            cases = [c for c in want['cases'] if c['period'] == period]
            deps = [{(ns, pod): off for ns, pod, off in c['departures']} for c in cases]
            sched, k8s, _ = mirror_session(script, factory)
            try:
                state, traffic = dict(sched.pod_state), k8s.transcript()
                before = {nd: (v.busy_time, list(v.pod_info), [x.pods_used for x in v.nics]) for nd, v in sched.nodes.items()}
                got = sched.ForecastDepartures(deps, SCANS, keys=keys, period=period, reasons=True)
                assert len(got) == len(cases)
                for c, d, (placement, reasons) in zip(cases, deps, got):
                    want_p = [None if p is None else (p[0], p[1]) for p in c['placed']]
                    assert list(placement) == keys and list(placement.values()) == want_p, (name, c['departures'])
                    assert reasons == _counted(c['reasons'], list(sched.nodes)), (name, c['departures'])
                    if n % 4 == 0:
                        assert sched.ForecastPending(SCANS, keys=keys, period=period, reasons=True,
                                                     departures=d) == (placement, reasons), name
                    n += 1
                assert k8s.transcript() == traffic and sched.pod_state == state, name
                assert {nd: (v.busy_time, list(v.pod_info), [x.pods_used for x in v.nics])
                        for nd, v in sched.nodes.items()} == before, name
            finally:
                sched.close()
    from tests.golden.make_departures_golden import departure_sessions, evidence
    golden = make_live_golden.load('departures')['sessions']
    assert [g['name'] for g in golden] == [name for name, _ in departure_sessions()] and all(evidence(golden))
    for (name, script), want in list(zip(departure_sessions(), golden))[:limit]:
        keys, cases = [tuple(k) for k in want['pending']], want['cases']
        sched, k8s, _ = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()
            cands = candidates(sched, cases, sched._node_cls)
            deps = [{(ns, pod): off for ns, pod, off in c['departures']} for c in cases]
            got = sched.ForecastDepartures(deps, SCANS, keys=keys, period=cases[0]['period'],
                                           additions=[c for c, _ in cands], reasons=True)
            for c, (placement, reasons), (_, grown) in zip(cases, got, cands):
                want_p = [None if p is None else (p[0], p[1]) for p in c['placed']]
                assert list(placement.values()) == want_p, (name, c['schedule'], bool(c['nodes']))
                assert reasons == _counted(c['reasons'], grown), (name, c['schedule'], bool(c['nodes']))
                n += 1
            assert k8s.transcript() == traffic and sched.pod_state == state, name
        finally:
            sched.close()
    golden = make_live_golden.load('forecast')['sessions']
    for (name, script), want in list(zip(forecast_sessions(), golden))[:limit]:
        keys = [tuple(k) for k in want['pending']]
        period, frac = VARIANTS[0]
        cases = [c for c in want['cases'] if (c['period'], c['frac']) == (period, frac)]
        if not cases:
            continue
        sched, k8s, clock = mirror_session(script, factory)
        try:
            clock.t += frac
            cands = candidates(sched, cases, sched._node_cls)
            got = sched.ForecastDepartures([{}] * len(cases), F_SCANS, keys=keys, period=period,
                                           additions=[c for c, _ in cands], reasons=True)
            for c, (placement, reasons), (_, grown) in zip(cases, got, cands):
                want_p = [None if p is None else (p[0], p[1]) for p in c['placed']]
                assert list(placement.values()) == want_p, (name, c['label'])
                assert reasons == _counted(c['reasons'], grown), (name, c['label'])
                n += 1
            assert got == sched.ForecastPending(F_SCANS, keys=keys, period=period, additions=[c for c, _ in cands],
                                                reasons=True), name
        finally:
            sched.close()
    assert limit is not None or n >= 250, n


def test_forecast_departures_equals_the_reference():
    """Several departure schedules of one session side by side, with and without an added node, and candidate nodes
    with empty schedules, with the oracle standing in for the device."""
    _schedules_against_the_reference(DeparturesPlanner)


def test_forecast_departures_checks_its_arguments():
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import release_sessions
    name, script = release_sessions()[-1]
    sched, _, _ = mirror_session(script, DeparturesPlanner)
    try:
        pending = list(sched.ForecastPending(3))
        deployed = [(ns, pod) for n in sched.nodes.values() for (pod, ns) in n.pod_info]
        # ForecastPending keeps refusing departures with additions: that combination is ForecastDepartures'
        with pytest.raises(ValueError):
            sched.ForecastPending(3, departures={deployed[0]: 10.0}, additions=[[]])
        for bad in ({pending[0]: 10.0}, {deployed[0]: 0.0}, {('ns0', 'never-annotated'): 10.0}):
            with pytest.raises(ValueError):
                sched.ForecastDepartures([{}, bad], 3)
        with pytest.raises(ValueError):
            sched.ForecastDepartures([{}, {}], 3, additions=[[]])
        assert sched.ForecastDepartures([], 3) == []
        d = {deployed[0]: 15.0}
        both = sched.ForecastDepartures([d, {}], 3, reasons=True)
        assert both[0] == sched.ForecastPending(3, departures=d, reasons=True)
        assert both[1] == sched.ForecastPending(3, reasons=True)
        assert both[0] != both[1]
    finally:
        sched.close()


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_departures_equal_the_oracle_in_every_sweep_mode():
    from nhd_b200.solver import Solver
    from tests.test_query import MODES
    tot, cuts = [0, 0], 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::6] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        calls = departure_calls(recs, speed, pods, now, busy, 100 + j)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s = Solver(speed, min_busy_secs=busy, **mode)
            try:
                tot = [a + b for a, b in zip(tot, check_calls(s, calls, speed, busy, (j, mode)))]
                if j % 4 == 0:
                    cuts += check_identities(s, calls, release_cases(recs, speed, pods, now, busy, 100 + j), speed, busy)
                if j == 1 and not mode:
                    check_refusals(s, *calls[3], speed, busy)
            finally:
                s.close()
    assert tot[0] > (100 if EMULATED else 2000) and tot[1] > 0 and cuts > 0, (tot, cuts)


@pytest.mark.gpu
def test_forecast_departures_on_the_gpu():
    from tests.test_plan import _gpu_factory
    _schedules_against_the_reference(_gpu_factory(), limit=3 if EMULATED else None)


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After config 4's solve, 256 departure schedules of 1 to 64 releases of placed pods (one or two pairings per
    claimed NIC, so some counters go to -1), each with its own 128 pending one-GPU pods (twice the nodes that can take
    them) over 8 scans, in one call on the mirror and one on the snapshot: both agree, 8 sampled scenarios equal the oracle, and every scenario equals
    ``nhd_plan_batch_releases`` of its own pods and releases."""
    import workload
    from nhd_b200.solver import Solver
    from tests.test_forecast import _steps
    from tests.test_forecast_batch import config4_pending
    recs, speed, pods, now = workload.make_workload(4)
    recs, tail = config4_pending(recs, pods, 4096, 64)
    rng = np.random.default_rng(44)
    s = Solver(speed, min_busy_secs=30.0)
    try:
        s.load_nodes(recs)
        b0 = s.solve_batch(pods, now)
        after = s.read_nodes()
        s.snapshot()
        t = float(now.max()) + 5.0
        rounds = _steps(t, 30.0, 8)
        placed = np.flatnonzero(b0['status'] == wire.PLACED)
        scs = []
        for k in range(256):
            n_rel = 1 + k % 64
            pick = rng.choice(placed, n_rel, replace=False)
            rels = []
            for q, i in enumerate(pick):
                rnd = 1 + q % len(rounds)
                lo = t if rnd == 1 else rounds[rnd - 2]
                rels.append(release_of(b0[i], pods[i], int(b0[i]['node']), rnd, lo + 0.5 * (rounds[rnd - 1] - lo),
                                       1 + int(rng.integers(2))))
            rels = np.array(sorted(rels, key=lambda x: (int(x['round']), float(x['clock']))), dtype=wire.RELEASE_DTYPE)
            tracked = sorted({int(x['node']) for x in rels})
            used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
            for q, node in enumerate(tracked):
                nn = int(after['n_nics'][node])
                used[q, :nn] = [int(after['nic_inuse'][node]) >> i & 1 for i in range(nn)]
            p = tail[np.sort(rng.choice(len(tail), 128, replace=False))]
            scs.append(Scenario((), p, np.full(len(p), t), None, None, None, rounds, (tracked, used, rels)))
        got = s.plan_scenarios(scs)
        snap = s.plan_scenarios(scs, source='snapshot')
        later = 0
        for k, ((code, pod, b, rnd), (c2, _, b2, r2), sc) in enumerate(zip(got, snap, scs)):
            assert code == 0 and c2 == 0 and b.tobytes() == b2.tobytes() and (rnd == r2).all(), k
            want, wrnd = s.plan_batch_releases(sc.pods, sc.now, rounds, *sc.releases)
            assert b.tobytes() == want.tobytes() and (rnd == wrnd).all(), (k, helpers.first_binding_diff(want, b))
            later += int(((b['status'] == wire.PLACED) & (rnd >= 1)).sum())
        for k in rng.choice(len(scs), 8, replace=False):
            wb, wrnd, _, _ = oracle_scenario_releases(after, speed, scs[k], busy=30.0)
            assert got[k][2].tobytes() == wb.tobytes() and (got[k][3] == wrnd).all(), \
                (int(k), helpers.first_binding_diff(wb, got[k][2]))
        assert later > 0
    finally:
        s.close()
