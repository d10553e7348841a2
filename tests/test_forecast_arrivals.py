"""Forecasts with pods created between the scans (``nhd_plan_scenarios_arrivals``, ``Solver.plan_scenarios`` with
``Scenario.arrive``, ``NHDScheduler.ForecastArrivals``).

The contract is ``nhd_plan_scenarios_releases`` with each later pod first attempted alone at its own clock, in its gap,
merged by clock with that gap's releases, and retried at every scan from then on: byte for byte each pod's placing or
last attempt, the round and the clock of that attempt, and the reasons of the pods whose last attempt found no node.
``oracle_scenario_arrivals`` (tests/arrivals_oracle.py) is that plan, one oracle solve per attempt.  The chain of
evidence:
  * on the CPU emulation of the device (tests/emu), both lane orders, seeded calls that mix round-0 pods with arrivals
    in several gaps (at a gap's start, at a scan's clock, at a release's clock), edits, additions, exclusions held and
    lifted, releases, negative counters and none, with and without reasons, equal that oracle; both identities of the
    header hold; every malformed argument is refused and nothing of the handle moves;
  * ``ForecastArrivals`` equals ``ForecastDepartures`` without arrivals on the release sessions, keeps the retry order
    and reads only, checks its arguments, and answers on the device as with the oracle standing in;
  * on the GPU the same cases in every sweep mode, and config 4 at full size after its solve (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import _lib, wire
from nhd_b200.solver import Scenario
from tests import helpers
from tests.arrivals_oracle import ArrivalsPlanner, oracle_scenario_arrivals
from tests.test_forecast_releases import release_cases, release_of
from tests.test_plan import _emu_lib
from tests.test_query import _filter_words, _gpu_cases, emu_cases, packed
from tests.test_sharded_ranks import emu_env  # noqa: F401  (the emulated two-rank environment, a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def test_the_symbol_is_declared_and_exported():
    from nhd_b200 import build
    build.build()
    text = open(os.path.join(ROOT, 'include', 'nhd_b200.h')).read()
    assert 'int32_t nhd_plan_scenarios_arrivals(nhd_handle* h, int32_t source, int32_t n_scenarios' in text
    assert 'nhd_plan_scenarios_arrivals' in _lib.EXPORTS and hasattr(_lib.load(), 'nhd_plan_scenarios_arrivals')


# ---------------------------------------------------------------------------------------------- the cases
def timeline(rng, p, c, rounds, rels, t0, n0=None):
    """``(pods, clocks, arrive, n0)``: the first ``n0`` pods (random when None) pending at their clocks, the rest
    arriving in random gaps, each at the gap's start, at its scan's clock, at one of its releases' clocks, mid-gap or at
    random inside it; pods reordered so that ``(arrive, clock)`` never goes down."""
    n = len(p)
    n0 = int(rng.integers(0, n + 1)) if n0 is None else min(n0, n)
    c = np.asarray(c, dtype='<f8').copy()
    first = float(c[:n0].max()) if n0 else t0
    ev = []
    for _ in range(n - n0):
        g = int(rng.integers(1, len(rounds) + 1))
        lo, hi = (first if g == 1 else rounds[g - 2]), rounds[g - 1]
        mine = [float(x) for x in rels['clock'][rels['round'] == g]] if len(rels) else []
        opts = [lo, hi, 0.5 * (lo + hi), lo + float(rng.random()) * (hi - lo)] + mine
        ev.append((g, opts[int(rng.integers(len(opts)))]))
    order = sorted(range(n - n0), key=lambda k: ev[k])
    idx = np.concatenate([np.arange(n0), n0 + np.asarray(order, dtype=np.int64)]).astype(np.int64)
    arrive = np.asarray([0] * n0 + [ev[k][0] for k in order], dtype='<i4')
    clock = np.concatenate([c[:n0], np.asarray([ev[k][1] for k in order], dtype='<f8')])
    return p[idx], clock, arrive, n0


def arrival_calls(recs, speed, pods, now, busy, seed):
    """``(state, [Scenario])`` calls on one stream, from ``release_cases``: per release case with rounds one call of
    nine scenarios on its state, each a random run of the pending pods with a random timeline: the case's releases
    alone, with an exclusion held throughout or lifted at a pod of round 0, with an edited node (its fresh record),
    with an added node (a copy of a fresh record), tracking without releases, no releases at all, every pod arriving
    (none pending at the start), and no arrivals."""
    rng = np.random.default_rng(2000 + seed)
    out = []
    for st, tail, clock, rounds, tracked, used, rels in release_cases(recs, speed, pods, now, busy, seed):
        if not len(tail) or not len(rounds):
            continue
        n = len(st)
        t0 = float(np.max(clock))
        rel_nodes = {int(x) for x in rels['node']}
        free = [k for k in range(n) if k not in rel_nodes and k not in tracked]
        full = (tracked, used, rels)

        def pick(r=rels, n0=None):
            k = int(rng.integers(1, min(len(tail), 10) + 1))
            idx = np.sort(rng.choice(len(tail), k, replace=False))
            return timeline(rng, tail[idx], clock[idx], rounds, r, t0, n0)
        p, c, a, _ = timeline(rng, tail, clock, rounds, rels, t0)
        scs = [Scenario((), p, c, None, None, None, rounds, full, a)]
        p, c, a, _ = pick()
        scs.append(Scenario([int(rng.integers(n))], p, c, None, None, None, rounds, full, a))
        p, c, a, n0 = pick()
        scs.append(Scenario([int(rng.integers(n))], p, c, int(rng.integers(n0 + 1)), None, None, rounds, full, a))
        if free:
            e = int(rng.choice(free))
            p, c, a, _ = pick()
            scs.append(Scenario((), p, c, None, ([e], recs[[e]]), None, rounds, full, a))
        p, c, a, _ = pick()
        k = int(rng.integers(n))
        scs.append(Scenario((), p, c, None, None, ([int(rng.integers(n + 1))], recs[[k]]), rounds, full, a))
        p, c, a, _ = pick(rels[:0])
        scs.append(Scenario((), p, c, None, None, None, rounds, (tracked, used, rels[:0]), a))
        p, c, a, _ = pick(rels[:0])
        scs.append(Scenario((), p, c, None, None, None, rounds, None, a))
        p, c, a, _ = pick(n0=0)
        scs.append(Scenario((), p, c, None, None, None, rounds, full, a))
        p, c, a, _ = pick(n0=len(tail))
        scs.append(Scenario((), p, c, None, None, None, rounds, full, None))
        out.append((st, scs))
    return out


def oracle_call(st, speed, scs, busy, explain):
    """Per scenario ``(bindings, pod_round, counts, pod_clock)`` of the oracle, added nodes numbered across the call."""
    res, base = [], 0
    for sc in scs:
        res.append(oracle_scenario_arrivals(st, speed, sc, base, busy, explain=explain))
        base += 0 if sc.adds is None else len(sc.adds[0])
    return res


def check_calls(s, calls, speed, busy, where=''):
    """Every call equals the oracle on every scenario, with reasons and without.  Returns (pods compared, arrivals
    placed on creation, arrivals placed at a later scan)."""
    n = created = later = 0
    for j, (st, scs) in enumerate(calls):
        s.load_nodes(st)
        got = s.plan_scenarios(scs, explain=True)
        plain = s.plan_scenarios(scs)
        want = oracle_call(st, speed, scs, busy, True)
        for k, ((code, pod, b, rows, rnd, clk), (wb, wrnd, wrows, wclk), sc, pl) in enumerate(zip(got, want, scs, plain)):
            assert code == 0, (where, j, k, code, pod)
            assert b.tobytes() == wb.tobytes(), (where, j, k, helpers.first_binding_diff(wb, b))
            assert (rnd == wrnd).all(), (where, j, k, rnd, wrnd)
            assert clk.tobytes() == wclk.tobytes(), (where, j, k, clk, wclk)
            assert (rows == wrows).all(), (where, j, k, np.flatnonzero((rows != wrows).any(1)))
            assert pl[2].tobytes() == b.tobytes() and (pl[3] == rnd).all() and pl[4].tobytes() == clk.tobytes()
            n += len(b)
            if sc.arrive is not None:
                arr = np.asarray(sc.arrive) > 0
                placed = arr & (b['status'] == wire.PLACED)
                on = placed & (clk == np.asarray(sc.now))
                created += int(on.sum())
                later += int((placed & ~on).sum())
    return n, created, later


class _ViaArrivals:
    """A library whose ``nhd_plan_scenarios_releases`` is ``nhd_plan_scenarios_arrivals`` with a NULL arrive_round:
    ``Solver.plan_scenarios`` through it tests the first identity of the header.  The pod clocks of the last call are
    kept in ``clocks``."""
    def __init__(self, L):
        self._L, self.clocks = L, None

    def __getattr__(self, name):
        return getattr(self._L, name)

    def nhd_plan_scenarios_releases(self, *a):
        import ctypes
        n = ctypes.cast(a[12], ctypes.POINTER(ctypes.c_int32))[a[2]]          # pod_start[n_scenarios]
        self.clocks = np.full(max(n, 1), np.nan, dtype='<f8')
        return self._L.nhd_plan_scenarios_arrivals(*a[:22], None, *a[22:], self.clocks.ctypes.data)


def _gap1_start(sc):
    """The latest clock a pod pending at the start of ``sc`` may have: its first round's, or the earliest release of
    that round."""
    rl = None if sc.releases is None else sc.releases[2]
    first = [] if rl is None else [float(c) for c in rl['clock'][rl['round'] == 1]]
    return min([float(sc.rounds[0])] + first)


def check_identities(s, calls):
    """A NULL arrive_round: ``nhd_plan_scenarios_releases`` byte for byte, reasons included, the pod clocks those of
    the pods' last attempts.  A scenario whose pods all arrive in gap 1 with no release of round 1: the releases
    call on the same pods as round-0 pods, its rounds with 0 read as 1.  Returns the scenarios compared."""
    n = 0
    for st, scs in calls:
        s.load_nodes(st)
        plain = [Scenario(*sc[:8])._replace(now=np.minimum(sc.now, _gap1_start(sc))) for sc in scs]   # all at the start
        a = s.plan_scenarios(plain, explain=True)
        L = s._L
        s._L = via = _ViaArrivals(L)
        try:
            b = s.plan_scenarios(plain, explain=True)
        finally:
            s._L = L
        assert all(x[:2] == y[:2] and all(u.tobytes() == v.tobytes() for u, v in zip(x[2:], y[2:])) for x, y in zip(a, b))
        at = 0
        for sc, (code, _, _, _, rnd) in zip(plain, a):
            clocks = np.asarray([sc.now[i] if r == 0 else sc.rounds[r - 1] for i, r in enumerate(rnd.tolist())])
            assert via.clocks[at:at + len(rnd)].tobytes() == clocks.tobytes()
            at += len(rnd)
        # the second identity
        ones = []
        for sc in plain:
            order = np.argsort(np.asarray(sc.now), kind='stable')
            tr, used, rl = sc.releases or ((), np.zeros((0, wire.MAX_NICS), dtype='<i2'), None)
            rl = None if rl is None else rl[rl['round'] != 1]
            lift = None if sc.lift is None else 0
            now = np.minimum(np.asarray(sc.now)[order], sc.rounds[0])        # every pod inside gap 1
            ones.append(Scenario(sc.exclude, sc.pods[order], now, lift, sc.edits, sc.adds,
                                 sc.rounds, None if sc.releases is None else (tr, used, rl)))
        rel = s.plan_scenarios([sc._replace(releases=sc.releases or ((), np.zeros((0, wire.MAX_NICS), dtype='<i2'),
                                                                      None)) for sc in ones], explain=True)
        arr = s.plan_scenarios([sc._replace(arrive=np.ones(len(sc.pods), dtype='<i4')) for sc in ones], explain=True)
        for x, y, sc in zip(rel, arr, ones):
            assert x[0] == 0 and y[0] == 0
            assert x[2].tobytes() == y[2].tobytes(), helpers.first_binding_diff(x[2], y[2])
            assert (x[3] == y[3]).all() and (np.maximum(x[4], 1) == y[4]).all()
            want = np.asarray([sc.now[i] if r == 0 else sc.rounds[r - 1] for i, r in enumerate(x[4].tolist())])
            assert y[5].tobytes() == want.tobytes()
            n += 1
    return n


def check_refusals(s, st, scs, speed, busy):
    """Every malformed arrival argument is NHD_ERR_INVALID and leaves records, snapshot, staged batch, bindings,
    bitmaps, explanations, timing and counters as they were; a plan afterwards equals one on a fresh handle."""
    from nhd_b200.solver import Solver, SolverError
    sc = next(x for x in scs if x.arrive is not None and (np.asarray(x.arrive) > 0).sum() >= 2
              and (np.asarray(x.arrive) == 0).sum() >= 2)
    other = scs[-1]
    rounds, arrive, now = list(sc.rounds), np.asarray(sc.arrive), np.asarray(sc.now)
    s.load_nodes(st)
    s.snapshot()
    b = s.solve_batch(sc.pods, sc.now)
    timing, counters = s.timing(), s.debug_counters()

    def state():
        words, pt = _filter_words(s)
        return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                s.explain_batch().tobytes())
    before = state()

    def refused(what, bad):
        with pytest.raises(SolverError) as e:
            s.plan_scenarios([other, bad], source='snapshot')
        assert e.value.code == wire.ERR_INVALID and what in str(e.value), (what, str(e.value))

    def arr(f):
        a = arrive.copy()
        f(a)
        return sc._replace(arrive=a)

    def clk(f):
        c = now.copy()
        f(c)
        return sc._replace(now=c)
    last = len(rounds)
    k = int(np.flatnonzero(arrive > 0)[0])                     # the first arrival
    refused('outside [0,', arr(lambda a: a.__setitem__(-1, last + 1)))
    refused('outside [0,', arr(lambda a: a.__setitem__(0, -1)))
    refused('go down', arr(lambda a: a.__setitem__(0, 1)))                # pod 1 is pending at the start
    refused('without rounds', sc._replace(rounds=None, releases=None))
    g = int(arrive[k])
    same = np.flatnonzero(arrive == g)
    if len(same) >= 2:
        refused('clocks go down', clk(lambda c: c.__setitem__(same[1], c[same[0]] - 1e-3)))
    lo = rounds[g - 2] if g > 1 else float(now[arrive == 0].max())
    refused('outside the gap', clk(lambda c: c.__setitem__(k, lo - 1.0)))
    refused('outside the gap', clk(lambda c: c.__setitem__(k, rounds[g - 1] + 1.0)))
    n0 = int((arrive == 0).sum())
    refused('lift index', sc._replace(lift=n0 + 1))
    assert state() == before
    assert s.timing() == timing and (s.debug_counters() == counters).all()
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


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
from nhd_b200.solver import Solver
from tests.test_forecast_arrivals import arrival_calls, check_calls, check_identities, check_refusals
from tests.test_query import emu_cases, packed
tot = [0] * 4
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        calls = arrival_calls(recs, speed, pods, now, busy, j)
        tot[:3] = [a + b for a, b in zip(tot, check_calls(s, calls, speed, busy, j))]
        if j %% 3 == 0:
            tot[3] += check_identities(s, calls)
        if j == 1:
            check_refusals(s, *calls[1], speed, busy)
    finally:
        s.close()
print('compared', *tot)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_arrivals_on_the_emulated_device_equal_the_oracle(lane_order):
    """``emu_cases()`` streams, half deployed: calls mixing round-0 pods with arrivals in several gaps, edits,
    additions, exclusions held and lifted, releases, negative starting counters, tracking alone and no releases, with
    reasons and without; both identities; the refusals."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=2400)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    n, created, later, ident = (int(x) for x in res.stdout.split()[-4:])
    assert n > 300 and created > 10 and later > 10 and ident > 10, res.stdout


# ---------------------------------------------------------------------------------------------- the scheduler
def _copies(sched, keys, rng, n, offs):
    """``n`` arrivals copying the configs and node groups of the pods ``keys`` (as their config maps hold them), named
    ``arrival-<k>``, each at a random offset: a scan's own, mid-gap, or just after the first scan."""
    from nhd_b200.NHDScheduler import Arrival
    out = []
    for k in range(n):
        ns, name = keys[int(rng.integers(len(keys)))][:2]
        _, cfgstr = sched.k8s.GetCfgMap(name, ns)
        g = int(rng.integers(1, len(offs)))
        at = (offs[g], 0.5 * (offs[g - 1] + offs[g]), offs[g - 1] + 0.25)[int(rng.integers(3))]
        out.append(Arrival((ns, f'arrival-{k}'), sched.k8s.GetCfgType(name, ns), cfgstr,
                           list(sched.k8s.GetPodNodeGroups(name, ns)), at))
    return out


def _sessions_against_departures(factory, limit=None):
    """On the release sessions: ``ForecastArrivals`` with empty arrival lists is ``ForecastDepartures`` with each scan
    read as its offset.  With arrivals, the pending pods come first and the arrivals after them in the given order; a
    pending pod placed by the first scan keeps its answer (nothing arrives before that scan); an arrival is placed at
    its own offset or at a scan's; and nothing is written.  Returns the arrivals placed."""
    from tests.golden import make_live_golden
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import SCANS, release_sessions
    rng = np.random.default_rng(7)
    placed = 0
    golden = make_live_golden.load('releases')['sessions']
    for (name, script), want in list(zip(release_sessions(), golden))[:limit]:
        keys = [tuple(k) for k in want['pending']]
        period = want['cases'][0]['period']
        deps = [{(ns, pod): off for ns, pod, off in c['departures']} for c in want['cases'] if c['period'] == period]
        offs = [period * k for k in range(SCANS)]
        sched, k8s, _ = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()
            before = {nd: (v.busy_time, list(v.pod_info), [x.pods_used for x in v.nics]) for nd, v in sched.nodes.items()}
            dep = sched.ForecastDepartures(deps, SCANS, keys=keys, period=period, reasons=True)
            got = sched.ForecastArrivals([[] for _ in deps], SCANS, keys=keys, period=period, departures=deps,
                                         reasons=True)
            for (p, why), (q, why2) in zip(dep, got):
                assert why == why2, name
                assert {k: None if v is None else (offs[v[0]], v[1]) for k, v in p.items()} == q, name
            arr = [_copies(sched, keys, rng, int(rng.integers(1, 6)), offs) for _ in deps]
            res = sched.ForecastArrivals(arr, SCANS, keys=keys, period=period, departures=deps)
            for a, q, (p, _) in zip(arr, res, got):
                assert list(q) == [(k[0], k[1]) for k in keys] + [x.key for x in a], name
                for k, v in p.items():
                    if v is not None and v[0] == 0.0:
                        assert q[k] == v, (name, k)
                for x in a:
                    v = q[x.key]
                    placed += v is not None
                    assert v is None or v[0] >= x.at or v[0] in offs, (name, x, v)
            assert k8s.transcript() == traffic and sched.pod_state == state, name
            assert {nd: (v.busy_time, list(v.pod_info), [x.pods_used for x in v.nics])
                    for nd, v in sched.nodes.items()} == before, name
        finally:
            sched.close()
    return placed


def _against_the_reference(factory, limit=None):
    """``ForecastArrivals`` with every case of a session in one call equals the unmodified reference's ``run()`` with
    those pods created and those deployed pods deleted between its scans, with the added node or none
    (tests/golden/live/arrivals.json.gz): for every pending and arriving pod the offset of its placing attempt and its
    node, and the reference's reasons at the last attempt of those never placed; nothing is written.  Returns the cases
    compared."""
    from nhd_b200.NHDScheduler import Arrival
    from tests.golden import make_live_golden
    from tests.golden.make_arrivals_golden import PERIOD, arrival_sessions, evidence
    from tests.golden.make_expand_golden import candidates
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import SCANS
    from tests.test_plan_reasons import _counted
    golden = make_live_golden.load('arrivals')['sessions']
    assert [g['name'] for g in golden] == [name for name, _ in arrival_sessions()] and all(evidence(golden))
    n = 0
    for (name, script), want in list(zip(arrival_sessions(), golden))[:limit]:
        keys, cases = [tuple(k) for k in want['pending']], want['cases']
        if not cases:
            continue
        sched, k8s, _ = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()
            cands = candidates(sched, cases, sched._node_cls)
            arrs = []
            for c in cases:
                arr = []
                for ns, pod, (lns, lpod), at in c['arrivals']:
                    _, cfgstr = k8s.GetCfgMap(lpod, lns)
                    arr.append(Arrival((ns, pod), k8s.GetCfgType(lpod, lns), cfgstr,
                                       list(k8s.GetPodNodeGroups(lpod, lns)), at))
                arrs.append(arr)
            deps = [{(ns, pod): off for ns, pod, off in c['departures']} for c in cases]
            got = sched.ForecastArrivals(arrs, SCANS, keys=keys, period=PERIOD, departures=deps,
                                         additions=[c for c, _ in cands], reasons=True)
            for c, (placement, reasons), (_, grown) in zip(cases, got, cands):
                want_p = [None if p is None else (p[0], p[1]) for p in c['placed']]
                where = (name, c['schedule'], c['set'], bool(c['nodes']))
                assert list(placement) == [(k[0], k[1]) for k in keys] + [(a[0], a[1]) for a in c['arrivals']], where
                assert list(placement.values()) == want_p, where
                assert reasons == _counted(c['reasons'], grown), where
                n += 1
            assert k8s.transcript() == traffic and sched.pod_state == state, name
        finally:
            sched.close()
    return n


def test_forecast_arrivals_equals_the_reference():
    """With the oracle standing in for the device."""
    assert _against_the_reference(ArrivalsPlanner) >= 250


def test_forecast_arrivals_without_arrivals_is_forecast_departures():
    """With the oracle standing in for the device."""
    assert _sessions_against_departures(ArrivalsPlanner) > 0


def test_forecast_arrivals_checks_its_arguments():
    from nhd_b200.NHDScheduler import Arrival
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import release_sessions
    name, script = release_sessions()[-1]
    sched, _, _ = mirror_session(script, ArrivalsPlanner)
    try:
        keys = sched._pending_keys()
        pending = list(sched.ForecastPending(3))
        deployed = [(ns, pod) for n in sched.nodes.values() for (pod, ns) in n.pod_info]
        ns, pod = pending[0]
        _, cfgstr = sched.k8s.GetCfgMap(pod, ns)
        cfgtype, groups = sched.k8s.GetCfgType(pod, ns), list(sched.k8s.GetPodNodeGroups(pod, ns))

        def arrival(key, at):
            return Arrival(key, cfgtype, cfgstr, groups, at)
        ok = arrival((ns, 'new-0'), 30.0)
        for bad in ([arrival(pending[0], 10.0)], [arrival(deployed[0], 10.0)], [ok, ok],
                    [arrival((ns, 'new-1'), 0.0)], [arrival((ns, 'new-1'), -1.0)], [arrival((ns, 'new-1'), 60.5)]):
            with pytest.raises(ValueError):
                sched.ForecastArrivals([[], bad], 3)
        with pytest.raises(ValueError):
            sched.ForecastArrivals([[ok]], 1)                          # one scan: no gap to arrive in
        with pytest.raises(ValueError):
            sched.ForecastArrivals([[ok], []], 3, departures=[{}])
        with pytest.raises(ValueError):
            sched.ForecastArrivals([[ok], []], 3, additions=[[]])
        with pytest.raises(ValueError):
            sched.ForecastArrivals([[ok]], 3, departures=[{pending[0]: 10.0}])
        assert sched.ForecastArrivals([], 3) == []
        # a config that does not parse maps to None, as for a pending pod
        broken = Arrival((ns, 'new-2'), cfgtype, '{not a config', groups, 30.0)
        got = sched.ForecastArrivals([[ok, broken]], 3, reasons=True)
        (placement, _), = got
        assert list(placement) == pending + [(ns, 'new-0'), (ns, 'new-2')] and placement[(ns, 'new-2')] is None
        assert len(keys) == len(pending)
    finally:
        sched.close()


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_arrivals_equal_the_oracle_in_every_sweep_mode():
    from nhd_b200.solver import Solver
    from tests.test_query import MODES
    tot, ident = [0, 0, 0], 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::6] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        calls = arrival_calls(recs, speed, pods, now, busy, 100 + j)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s = Solver(speed, min_busy_secs=busy, **mode)
            try:
                tot = [a + b for a, b in zip(tot, check_calls(s, calls, speed, busy, (j, mode)))]
                if j % 4 == 0:
                    ident += check_identities(s, calls)
                if j == 1 and not mode:
                    check_refusals(s, *calls[1], speed, busy)
            finally:
                s.close()
    assert tot[0] > (100 if EMULATED else 2000) and tot[1] > 0 and tot[2] > 0 and ident > 0, (tot, ident)


@pytest.mark.gpu
def test_forecast_arrivals_on_the_gpu():
    """The scheduler on the device equals the reference file, and answers as with the oracle standing in on the
    release sessions with copied arrivals."""
    from tests.test_plan import _gpu_factory
    assert _against_the_reference(_gpu_factory(), limit=3 if EMULATED else None) > 0
    assert _sessions_against_departures(_gpu_factory(), limit=3 if EMULATED else None) > 0
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import SCANS, release_sessions
    rng_a, rng_b = np.random.default_rng(9), np.random.default_rng(9)
    for name, script in release_sessions()[:3 if EMULATED else None]:
        res = []
        for factory, rng in ((ArrivalsPlanner, rng_a), (_gpu_factory(), rng_b)):
            sched, _, _ = mirror_session(script, factory)
            try:
                keys = sched._pending_keys()
                if not keys:
                    break
                arr = [_copies(sched, keys, rng, k, [30.0 * x for x in range(SCANS)]) for k in (1, 4, 9)]
                res.append(sched.ForecastArrivals(arr, SCANS, keys=keys, reasons=True))
            finally:
                sched.close()
        if len(res) == 2:
            assert res[0] == res[1], name


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After config 4's solve, 256 timelines of 1 to 64 one-GPU arrivals over 8 scans (every other one with
    departures of placed pods), each after its own 64 pending pods, in one call on the mirror and one on the snapshot:
    both agree, every timeline with no release of round 1 and no pending pod equals the second identity, and 8 sampled
    timelines equal the oracle."""
    import workload
    from nhd_b200.solver import Solver
    from tests.test_forecast import _steps
    from tests.test_forecast_batch import config4_pending
    recs, speed, pods, now = workload.make_workload(4)
    recs, tail = config4_pending(recs, pods, 4096, 64)
    rng = np.random.default_rng(45)
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
            n_arr = 1 + k % 64
            rels = np.zeros(0, dtype=wire.RELEASE_DTYPE)
            if k % 2:
                pick = rng.choice(placed, 8, replace=False)
                rl = []
                for q, i in enumerate(pick):
                    rnd = 2 + q % (len(rounds) - 1)
                    lo = rounds[rnd - 2]
                    rl.append(release_of(b0[i], pods[i], int(b0[i]['node']), rnd, lo + 0.5 * (rounds[rnd - 1] - lo),
                                         1 + int(rng.integers(2))))
                rels = np.array(sorted(rl, key=lambda x: (int(x['round']), float(x['clock']))), dtype=wire.RELEASE_DTYPE)
            tracked = sorted({int(x['node']) for x in rels})
            used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
            for q, node in enumerate(tracked):
                nn = int(after['n_nics'][node])
                used[q, :nn] = [int(after['nic_inuse'][node]) >> i & 1 for i in range(nn)]
            n0 = 0 if k % 4 < 2 else 64
            p = tail[np.sort(rng.choice(len(tail), n0 + n_arr, replace=False))]
            gaps = np.sort(rng.integers(1, len(rounds) + 1, n_arr)) if k % 8 >= 2 else np.ones(n_arr, dtype=np.int64)
            clock = np.full(n0 + n_arr, t)
            for q, g in enumerate(gaps):
                lo = t if g == 1 else rounds[g - 2]
                clock[n0 + q] = lo + (q + 1) / (n_arr + 1) * (rounds[g - 1] - lo)
            arrive = np.concatenate([np.zeros(n0, dtype='<i4'), gaps.astype('<i4')])
            order = np.lexsort((clock, arrive))
            scs.append(Scenario((), p[order], clock[order], None, None, None, rounds, (tracked, used, rels),
                                arrive[order]))
        got = s.plan_scenarios(scs)
        snap = s.plan_scenarios(scs, source='snapshot')
        ident = created = 0
        for k, ((code, pod, b, rnd, clk), (c2, _, b2, r2, k2), sc) in enumerate(zip(got, snap, scs)):
            assert code == 0 and c2 == 0 and b.tobytes() == b2.tobytes() and (rnd == r2).all(), k
            assert clk.tobytes() == k2.tobytes(), k
            a = np.asarray(sc.arrive)
            created += int(((b['status'] == wire.PLACED) & (a > 0) & (clk == np.asarray(sc.now))).sum())
            if (a == 1).all():
                (_, _, want, wrnd), = s.plan_scenarios([sc._replace(arrive=None)])
                assert b.tobytes() == want.tobytes() and (rnd == np.maximum(wrnd, 1)).all(), k
                wclk = np.where(wrnd == 0, np.asarray(sc.now), np.asarray(rounds)[np.maximum(wrnd, 1) - 1])
                assert clk.tobytes() == wclk.tobytes(), k        # the releases call's clock of each last attempt
                ident += 1
        for k in rng.choice(len(scs), 8, replace=False):
            wb, wrnd, _, wclk = oracle_scenario_arrivals(after, speed, scs[k], busy=30.0)
            assert got[k][2].tobytes() == wb.tobytes() and (got[k][3] == wrnd).all(), \
                (int(k), helpers.first_binding_diff(wb, got[k][2]))
            assert got[k][4].tobytes() == wclk.tobytes(), int(k)
        assert ident >= 16 and created > 0, (ident, created)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------- sharded ranks
RANK_WORKER = r'''
import ctypes, os, pickle, sys, time
import numpy as np
root, tmp, rank, world = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
sys.path.insert(0, root)
if world > 1:
    ctypes.CDLL(os.path.join(root, 'tests', 'emu', 'fake_nccl', 'libnccl.so.2'), mode=ctypes.RTLD_GLOBAL)
from nhd_b200.solver import Solver, nccl_unique_id
recs, speed, pods, now, scs = pickle.load(open(os.path.join(tmp, 'in.pkl'), 'rb'))
nid = None
if world > 1:
    idf = os.path.join(tmp, 'nccl_id')
    if rank == 0:
        nid = nccl_unique_id()
        open(idf + '.tmp', 'wb').write(nid); os.rename(idf + '.tmp', idf)
    else:
        t0 = time.time()
        while not os.path.exists(idf):
            time.sleep(0.02)
            assert time.time() - t0 < 120
        nid = open(idf, 'rb').read()
s = Solver(speed, rank=rank, world_size=world, nccl_id=nid)
s.load_nodes(recs)
b = s.solve_batch(pods, now)
res = None
if rank == world - 1:                        # the last rank alone: the other never makes this call
    res = s.plan_scenarios(scs, explain=True)
pickle.dump((b, s.read_nodes(), res), open(os.path.join(tmp, 'out%d_%d.pkl' % (world, rank)), 'wb'))
s.close()
print('rank', rank, 'done')
'''


def test_rank_local_arrivals_on_sharded_ranks(emu_env, tmp_path):
    """On emulated two-rank handles, after a sharded batch, one ``nhd_plan_scenarios_arrivals`` call made by one rank
    alone (no collective) equals the answer of a single-rank handle given the same records and batch, reasons, rounds
    and clocks included."""
    import pickle
    import workload
    env = emu_env
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=500, wild=True)
    rng = np.random.default_rng(31)
    t0 = float(now.max())
    rounds = [t0 + 30.0 * k for k in range(1, 5)]
    scs = []
    for k in range(6):
        p = pods[300 + 20 * k:300 + 20 * k + 16]
        n0 = 4 * (k % 3)
        arrive = np.concatenate([np.zeros(n0, dtype='<i4'), np.sort(rng.integers(1, 5, len(p) - n0)).astype('<i4')])
        clock = np.asarray([t0 if g == 0 else rounds[g - 1] - 30.0 + 1.0 + 0.5 * q for q, g in enumerate(arrive)])
        scs.append(Scenario([int(rng.integers(1800))], p, clock, None if k % 2 else 0, None, None, rounds, None, arrive))
    pickle.dump((recs, speed, pods[:300], now[:300], scs), open(tmp_path / 'in.pkl', 'wb'))
    outs = {}
    for world, extra in ((2, {'NHD_SHARD_MIN_PAIRS': '1'}), (1, {})):
        procs = [subprocess.Popen([sys.executable, '-c', RANK_WORKER, ROOT, str(tmp_path), str(r), str(world)],
                                  cwd=ROOT, env=dict(env, EMU_LANE_ORDER='ad'[r], **extra), stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True) for r in range(world)]
        logs = [p.communicate(timeout=900)[0] for p in procs]
        for r, (p, o) in enumerate(zip(procs, logs)):
            assert p.returncode == 0, (world, r, o[-3000:])
        outs[world] = [pickle.load(open(tmp_path / f'out{world}_{r}.pkl', 'rb')) for r in range(world)]
    (b1, f1, want), = outs[1]
    for b, f, _ in outs[2]:
        assert b.tobytes() == b1.tobytes() and f.tobytes() == f1.tobytes()
    got = outs[2][1][2]
    placed = 0
    for x, y in zip(got, want):
        assert x[:2] == y[:2] == (0, -1)
        assert all(u.tobytes() == v.tobytes() for u, v in zip(x[2:], y[2:]))
        placed += int((x[2]['status'] == wire.PLACED).sum())
    assert placed > 0
