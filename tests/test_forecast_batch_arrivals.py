"""Forecasts of one large timeline with pods created between the scans, on the batch path (``nhd_plan_batch_arrivals``,
``Solver.plan_batch_arrivals``, ``NHDScheduler.ForecastPending(arrivals=...)``).

The contract is ``nhd_plan_scenarios_arrivals`` with this one timeline as a scenario, exclusions held throughout, no
edits and no additions: byte for byte each pod's placing or last attempt, its round and clock, and the reasons of the
pods whose last attempt found no node.  ``oracle_scenario_arrivals`` (tests/arrivals_oracle.py) is that plan.  The batch
path is exact because (DESIGN §8.18) a run of arrivals between two releases is a batch at per-pod clocks, releases
split a gap into blocks, and every arrival of a gap comes after every survivor of the scan before it in pod order.
The chain of evidence:
  * on the CPU emulation of the device (tests/emu), both lane orders, seeded timelines with arrivals at a gap's start,
    mid-gap, at a scan's clock and at a release's clock, bursts at one clock, no round-0 pods, every pod in the last
    gap, a pod type found only among the arrivals, negative counters and two pairings per NIC (cuts inside arrival runs
    and scans), no, every third and every GPU node excluded, mirror and snapshot sources, with and without reasons,
    equal that oracle and the scenario call; both identities of the header hold; every malformed argument is refused
    and nothing of the handle moves;
  * on an emulated two-rank handle one rank alone makes the call;
  * ``ForecastPending(arrivals=...)`` equals the reference file without added nodes, with the oracle standing in and
    on the emulated device, equals ``ForecastArrivals([a])[0]`` and checks its arguments;
  * on the GPU the same comparisons in every sweep mode, and config 4 at full size (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import _lib, wire
from nhd_b200.solver import Scenario
from tests import helpers
from tests.arrivals_oracle import ArrivalsPlanner, oracle_scenario_arrivals
from tests.test_forecast_arrivals import timeline
from tests.test_forecast_releases import release_cases, release_of
from tests.test_plan import _emu_lib
from tests.test_query import _filter_words, _gpu_cases, packed
from tests.test_sharded_ranks import emu_env  # noqa: F401  (the emulated two-rank environment, a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def test_the_symbol_is_declared_and_exported():
    from nhd_b200 import build
    build.build()
    text = open(os.path.join(ROOT, 'include', 'nhd_b200.h')).read()
    assert 'int32_t nhd_plan_batch_arrivals(nhd_handle* h, int32_t source, int32_t n_excluded' in text
    assert 'nhd_plan_batch_arrivals' in _lib.EXPORTS and hasattr(_lib.load(), 'nhd_plan_batch_arrivals')


# ---------------------------------------------------------------------------------------------- the cases
def _burst(sc):
    """``sc`` with each gap's arrivals all at one clock: the gap's first arrival's (the constant-clock path)."""
    a, c = np.asarray(sc.arrive), np.asarray(sc.now, dtype='<f8').copy()
    for g in set(a[a > 0].tolist()):
        c[a == g] = c[a == g].min()
    return sc._replace(now=c)


def batch_timelines(recs, speed, pods, now, busy, seed):
    """``(state, [Scenario])`` per release case with rounds: single timelines, exclusions held throughout, no edits and
    no additions.  A random timeline with the case's releases; with every third node and with every GPU node excluded;
    bursts sharing a clock; no round-0 pods; every pod arriving in the last gap (releases of earlier gaps then meet no
    pending pod); a pod type found only among the arrivals (the round-0 pods all copies of one pod); tracking without
    releases; no tracking at all."""
    rng = np.random.default_rng(5000 + seed)
    out = []
    for st, tail, clock, rounds, tracked, used, rels in release_cases(recs, speed, pods, now, busy, seed):
        if not len(tail) or not len(rounds):
            continue
        n = len(st)
        t0 = float(np.max(clock))
        full = (tracked, used, rels)

        def tl(r=rels, n0=None, p=tail, c=clock):
            return timeline(rng, p, c, rounds, r, t0, n0)[:3]
        scs = []
        p, c, a = tl()
        scs.append(Scenario((), p, c, None, None, None, rounds, full, a))
        scs.append(Scenario(list(range(0, n, 3)), p, c, None, None, None, rounds, full, a))
        gpu = [int(k) for k in np.flatnonzero(st['n_gpus'] > 0)]
        scs.append(Scenario(gpu, p, c, None, None, None, rounds, full, a))
        scs.append(_burst(Scenario((), p, c, None, None, None, rounds, full, a)))
        p, c, a = tl(n0=0)
        scs.append(Scenario((), p, c, None, None, None, rounds, full, a))
        last = len(rounds)
        lo = t0 if last == 1 else rounds[-2]
        k = len(tail)
        c2 = np.sort(lo + rng.random(k) * (rounds[-1] - lo))
        scs.append(Scenario((), tail, c2, None, None, None, rounds, full, np.full(k, last, dtype='<i4')))
        if len(tail) >= 3:
            k0 = min(len(tail) - 1, 4)
            p2 = np.concatenate([tail[:1].repeat(k0), tail[1:]])
            c3 = np.concatenate([np.full(k0, t0), clock[1:]])
            p, c, a, = timeline(rng, p2, c3, rounds, rels, t0, k0)[:3]
            scs.append(Scenario((), p, c, None, None, None, rounds, full, a))
        p, c, a = tl(r=rels[:0])
        scs.append(Scenario((), p, c, None, None, None, rounds, (tracked, used, rels[:0]), a))
        scs.append(Scenario([int(rng.integers(n))], p, c, None, None, None, rounds, None, a))
        out.append((st, scs))
    return out


def _rel(sc):
    tr, used, rl = sc.releases or ((), np.zeros((0, wire.MAX_NICS), dtype='<i2'), None)
    return tr, used, rl


def batch(s, sc, source='mirror', explain=True, arrive=True):
    """``Solver.plan_batch_arrivals`` of one timeline: ``(bindings, pod_round, pod_clock, counts)``."""
    tr, used, rl = _rel(sc)
    a = sc.arrive if arrive else np.zeros(len(sc.pods), dtype='<i4')
    r = s.plan_batch_arrivals(sc.pods, sc.now, sc.rounds, tr, used, rl, a, source=source, exclude=sc.exclude,
                              explain=explain)
    return r if explain else r + (None,)


def check_timelines(s, calls, speed, busy, where='', oracle=None):
    """Every timeline equals the oracle and the scenario call, with reasons and without, on the mirror and (every other
    call) on the snapshot after the mirror moved on.  ``oracle``: a dict that keeps the oracle's answers across calls
    on the same timelines.  Returns (pods compared, arrivals placed on creation, arrivals placed at a later scan)."""
    n = created = later = 0
    oracle = {} if oracle is None else oracle
    for j, (st, scs) in enumerate(calls):
        s.load_nodes(st)
        source = 'mirror'
        if j % 2:
            s.snapshot()
            s.solve_batch(scs[0].pods[:2], np.full(2, float(np.min(scs[0].now))))
            source = 'snapshot'
        scen = s.plan_scenarios(scs, source=source, explain=True)
        for k, sc in enumerate(scs):
            b, rnd, clk, rows = batch(s, sc, source)
            pb, prnd, pclk, _ = batch(s, sc, source, explain=False)
            if (j, k) not in oracle:
                oracle[(j, k)] = oracle_scenario_arrivals(st, speed, sc, 0, busy, explain=True)
            wb, wrnd, wrows, wclk = oracle[(j, k)]
            at = (where, j, k)
            assert b.tobytes() == wb.tobytes(), (at, helpers.first_binding_diff(wb, b))
            assert (rnd == wrnd).all(), (at, rnd, wrnd)
            assert clk.tobytes() == wclk.tobytes(), (at, clk, wclk)
            assert (rows == wrows).all(), (at, np.flatnonzero((rows != wrows).any(1)))
            assert pb.tobytes() == b.tobytes() and (prnd == rnd).all() and pclk.tobytes() == clk.tobytes(), at
            code, _, sb, srows, srnd, sclk = scen[k]
            assert code == 0 and sb.tobytes() == b.tobytes() and (srnd == rnd).all(), at
            assert sclk.tobytes() == clk.tobytes() and (srows == rows).all(), at
            n += len(b)
            arr = np.asarray(sc.arrive) > 0
            placed = arr & (b['status'] == wire.PLACED)
            on = placed & (clk == np.asarray(sc.now))
            created += int(on.sum())
            later += int((placed & ~on).sum())
    return n, created, later


class _ViaArrivals:
    """A library whose ``nhd_plan_batch_releases`` is ``nhd_plan_batch_arrivals`` with a NULL arrive_round; the pod
    clocks of the last call are kept in ``clocks``."""
    def __init__(self, L):
        self._L, self.clocks = L, None

    def __getattr__(self, name):
        return getattr(self._L, name)

    def nhd_plan_batch_releases(self, *a):
        self.clocks = np.full(max(a[4], 1), np.nan, dtype='<f8')
        return self._L.nhd_plan_batch_arrivals(*a[:14], None, *a[14:], self.clocks.ctypes.data)


def check_identities(s, calls):
    """A NULL arrive_round: ``nhd_plan_batch_releases`` byte for byte, reasons included, the pod clocks those of the
    pods' last attempts; every case of ``release_cases`` is taken, those that cut included.  Returns the timelines
    compared."""
    n = 0
    for st, scs in calls:
        s.load_nodes(st)
        for sc in scs:
            tr, used, rl = _rel(sc)
            first = [] if rl is None else [float(c) for c in rl['clock'][rl['round'] == 1]]
            plain = sc._replace(now=np.minimum(np.asarray(sc.now), min([float(sc.rounds[0])] + first)))
            want = s.plan_batch_releases(plain.pods, plain.now, plain.rounds, tr, used, rl, exclude=plain.exclude,
                                         explain=True)
            L = s._L
            s._L = via = _ViaArrivals(L)
            try:
                got = s.plan_batch_releases(plain.pods, plain.now, plain.rounds, tr, used, rl, exclude=plain.exclude,
                                            explain=True)
            finally:
                s._L = L
            assert all(u.tobytes() == v.tobytes() for u, v in zip(got, want))
            rnd = want[1]
            clocks = np.asarray([plain.now[i] if r == 0 else plain.rounds[r - 1] for i, r in enumerate(rnd.tolist())])
            assert via.clocks[:len(rnd)].tobytes() == clocks.tobytes()
            n += 1
    return n


def check_refusals(s, st, scs, speed, busy):
    """Every malformed arrival argument is NHD_ERR_INVALID and leaves records, snapshot, staged batch, bindings,
    bitmaps, explanations, timing and counters as they were; a plan afterwards equals one on a fresh handle."""
    from nhd_b200.solver import Solver, SolverError
    sc = next(x for x in scs if (np.asarray(x.arrive) > 0).sum() >= 2 and (np.asarray(x.arrive) == 0).sum() >= 2)
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
            batch(s, bad, 'snapshot')
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
    k = int(np.flatnonzero(arrive > 0)[0])
    refused('outside [0,', arr(lambda a: a.__setitem__(-1, last + 1)))
    refused('outside [0,', arr(lambda a: a.__setitem__(0, -1)))
    refused('go down', arr(lambda a: a.__setitem__(0, 1)))
    refused('without rounds', sc._replace(rounds=[], releases=None))
    g = int(arrive[k])
    same = np.flatnonzero(arrive == g)
    if len(same) >= 2:
        refused('clocks go down', clk(lambda c: c.__setitem__(same[1], c[same[0]] - 1e-3)))
    lo = rounds[g - 2] if g > 1 else float(now[arrive == 0].max())
    refused('outside the gap', clk(lambda c: c.__setitem__(k, lo - 1.0)))
    refused('outside the gap', clk(lambda c: c.__setitem__(k, rounds[g - 1] + 1.0)))
    assert state() == before
    assert s.timing() == timing and (s.debug_counters() == counters).all()
    got = [batch(s, x, 'snapshot') for x in scs]
    assert state() == before
    fresh = Solver(speed, min_busy_secs=busy)
    try:
        fresh.load_nodes(st)
        want = [batch(fresh, x) for x in scs]
    finally:
        fresh.close()
    assert all(all(u.tobytes() == v.tobytes() for u, v in zip(x, y)) for x, y in zip(got, want))
    s.restore()
    s.solve_staged()
    assert s.fetch_bindings().tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
from nhd_b200.solver import Solver
from tests.test_forecast_batch_arrivals import batch_timelines, check_timelines, check_identities, check_refusals
from tests.test_query import emu_cases, packed
tot = [0] * 4
for j, scn in list(enumerate(emu_cases()))[::3]:
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        calls = batch_timelines(recs, speed, pods, now, busy, j)
        tot[:3] = [a + b for a, b in zip(tot, check_timelines(s, calls, speed, busy, j))]
        if j %% 2 == 0:
            tot[3] += check_identities(s, calls)
        if j == 3:
            check_refusals(s, *calls[1], speed, busy)
    finally:
        s.close()
print('compared', *tot)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_batch_arrivals_on_the_emulated_device_equal_the_oracle(lane_order):
    """Every third ``emu_cases()`` stream, half deployed: the timelines of ``batch_timelines`` against the oracle and the scenario
    call, with reasons and without, on the mirror and the snapshot; the first identity; the refusals."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=2400)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    n, created, later, ident = (int(x) for x in res.stdout.split()[-4:])
    assert n > 1000 and created > 10 and later > 10 and ident > 10, res.stdout


# ---------------------------------------------------------------------------------------------- the scheduler
class BatchArrivalsPlanner(ArrivalsPlanner):
    """``ArrivalsPlanner`` that also answers ``plan_batch_arrivals``, with ``oracle_scenario_arrivals`` on the one
    timeline, exclusions held.  TEST INFRASTRUCTURE."""

    def plan_batch_arrivals(self, pods, now, round_clocks, tracked, pods_used, releases, arrive_round,
                            source='mirror', exclude=(), explain=False):
        sc = Scenario(list(exclude), pods, now, None, None, None, list(round_clocks),
                      (tracked, pods_used, releases), arrive_round)
        b, rnd, counts, clock = oracle_scenario_arrivals(self._source(source), self._speed, sc, 0, self._min_busy,
                                                         explain=explain)
        return (b, rnd, clock, counts) if explain else (b, rnd, clock)


def _against_the_reference(factory, limit=None):
    """``ForecastPending(arrivals=...)`` per case without an added node equals the unmodified reference's ``run()``
    (tests/golden/live/arrivals.json.gz) on offsets, nodes and reasons, and equals ``ForecastArrivals([a])[0]``;
    nothing is written.  Returns the cases compared."""
    from nhd_b200.NHDScheduler import Arrival
    from tests.golden import make_live_golden
    from tests.golden.make_arrivals_golden import PERIOD, arrival_sessions
    from tests.golden.make_expand_golden import candidates
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import SCANS
    from tests.test_plan_reasons import _counted
    golden = make_live_golden.load('arrivals')['sessions']
    n = 0
    for (name, script), want in list(zip(arrival_sessions(), golden))[:limit]:
        keys, cases = [tuple(k) for k in want['pending']], [c for c in want['cases'] if not c['nodes']]
        if not cases:
            continue
        sched, k8s, _ = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()
            for c, (_, grown) in zip(cases, candidates(sched, cases, sched._node_cls)):
                arr = []
                for ns, pod, (lns, lpod), at in c['arrivals']:
                    _, cfgstr = k8s.GetCfgMap(lpod, lns)
                    arr.append(Arrival((ns, pod), k8s.GetCfgType(lpod, lns), cfgstr,
                                       list(k8s.GetPodNodeGroups(lpod, lns)), at))
                dep = {(ns, pod): off for ns, pod, off in c['departures']}
                placement, reasons = sched.ForecastPending(SCANS, keys=keys, period=PERIOD, reasons=True,
                                                           departures=dep, arrivals=arr)
                where = (name, c['schedule'], c['set'])
                assert list(placement) == [(k[0], k[1]) for k in keys] + [(a[0], a[1]) for a in c['arrivals']], where
                assert list(placement.values()) == [None if p is None else (p[0], p[1]) for p in c['placed']], where
                assert reasons == _counted(c['reasons'], grown), where
                assert (placement, reasons) == sched.ForecastArrivals([arr], SCANS, keys=keys, period=PERIOD,
                                                                      departures=[dep], reasons=True)[0], where
                n += 1
            assert k8s.transcript() == traffic and sched.pod_state == state, name
        finally:
            sched.close()
    return n


def test_forecast_pending_with_arrivals_equals_the_reference():
    """With the oracle standing in for the device."""
    assert _against_the_reference(BatchArrivalsPlanner) >= 100


EMU_SCHED_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
from tests.test_forecast_batch_arrivals import _against_the_reference
from tests.test_plan import _gpu_factory
print('compared', _against_the_reference(_gpu_factory(), limit=6))
'''


def test_forecast_pending_with_arrivals_on_the_emulated_device():
    """The scheduler on the emulated device, on the first sessions of the reference file."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1')
    res = subprocess.run([sys.executable, '-c', EMU_SCHED_CODE % dict(root=ROOT)], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=2400)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    assert int(res.stdout.split()[-1]) > 0, res.stdout


def test_forecast_pending_checks_its_arrivals():
    from nhd_b200.NHDScheduler import Arrival
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import release_sessions
    name, script = release_sessions()[-1]
    sched, _, _ = mirror_session(script, BatchArrivalsPlanner)
    try:
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
                sched.ForecastPending(3, arrivals=bad)
        with pytest.raises(ValueError):
            sched.ForecastPending(1, arrivals=[ok])                     # one scan: no gap to arrive in
        with pytest.raises(ValueError):
            sched.ForecastPending(3, arrivals=[ok], additions=[[]])
        with pytest.raises(ValueError):
            sched.ForecastPending(3, arrivals=[ok], departures={pending[0]: 10.0})
        assert sched.ForecastPending(3, arrivals=[]) == sched.ForecastArrivals([[]], 3)[0]
        got = sched.ForecastPending(3, arrivals=[ok], reasons=True)
        assert got == sched.ForecastArrivals([[ok]], 3, reasons=True)[0]
        assert list(got[0]) == pending + [(ns, 'new-0')]
        # without arrivals ForecastPending is as before: scans as ints
        assert all(p is None or isinstance(p[0], int) for p in sched.ForecastPending(3).values())
    finally:
        sched.close()


# ---------------------------------------------------------------------------------------------- sharded ranks
RANK_WORKER = r'''
import ctypes, os, pickle, sys, time
import numpy as np
root, tmp, rank, world = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
sys.path.insert(0, root)
if world > 1:
    ctypes.CDLL(os.path.join(root, 'tests', 'emu', 'fake_nccl', 'libnccl.so.2'), mode=ctypes.RTLD_GLOBAL)
from nhd_b200.solver import Solver, nccl_unique_id
recs, speed, pods, now, tls = pickle.load(open(os.path.join(tmp, 'in.pkl'), 'rb'))
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
    res = [s.plan_batch_arrivals(p, c, rounds, (), (), None, a, exclude=ex, explain=True) for p, c, rounds, a, ex in tls]
pickle.dump((b, s.read_nodes(), res), open(os.path.join(tmp, 'out%d_%d.pkl' % (world, rank)), 'wb'))
s.close()
print('rank', rank, 'done')
'''


def test_rank_local_batch_arrivals_on_sharded_ranks(emu_env, tmp_path):
    """On emulated two-rank handles, after a sharded batch, ``nhd_plan_batch_arrivals`` calls made by one rank alone
    (no collective) equal those of a single-rank handle given the same records and batch, reasons included."""
    import pickle
    import workload
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=500, wild=True)
    rng = np.random.default_rng(37)
    t0 = float(now.max())
    rounds = [t0 + 30.0 * k for k in range(1, 5)]
    tls = []
    for k in range(4):
        p = pods[300 + 40 * k:300 + 40 * k + 40]
        n0 = 10 * (k % 3)
        arrive = np.concatenate([np.zeros(n0, dtype='<i4'), np.sort(rng.integers(1, 5, len(p) - n0)).astype('<i4')])
        clock = np.asarray([t0 if g == 0 else rounds[g - 1] - 30.0 + 1.0 + 0.25 * q for q, g in enumerate(arrive)])
        tls.append((p, clock, rounds, arrive, [int(rng.integers(1800))] if k % 2 else []))
    pickle.dump((recs, speed, pods[:300], now[:300], tls), open(tmp_path / 'in.pkl', 'wb'))
    outs = {}
    for world, extra in ((2, {'NHD_SHARD_MIN_PAIRS': '1'}), (1, {})):
        procs = [subprocess.Popen([sys.executable, '-c', RANK_WORKER, ROOT, str(tmp_path), str(r), str(world)],
                                  cwd=ROOT, env=dict(emu_env, EMU_LANE_ORDER='ad'[r], **extra), stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True) for r in range(world)]
        logs = [p.communicate(timeout=900)[0] for p in procs]
        for r, (p, o) in enumerate(zip(procs, logs)):
            assert p.returncode == 0, (world, r, o[-3000:])
        outs[world] = [pickle.load(open(tmp_path / f'out{world}_{r}.pkl', 'rb')) for r in range(world)]
    (b1, f1, want), = outs[1]
    for b, f, _ in outs[2]:
        assert b.tobytes() == b1.tobytes() and f.tobytes() == f1.tobytes()
    placed = 0
    for x, y in zip(outs[2][1][2], want):
        assert all(u.tobytes() == v.tobytes() for u, v in zip(x, y))
        placed += int((x[0]['status'] == wire.PLACED).sum())
    assert placed > 0


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_batch_arrivals_equal_the_oracle_in_every_sweep_mode():
    from nhd_b200.solver import Solver
    from tests.test_query import MODES
    tot, ident = [0, 0, 0], 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::6]):
        recs, pods, now, speed, busy = packed(scn)
        calls = batch_timelines(recs, speed, pods, now, busy, 100 + j)
        oracle = {}
        for mode in (MODES[:1] if EMULATED else MODES):
            s = Solver(speed, min_busy_secs=busy, **mode)
            try:
                tot = [a + b for a, b in zip(tot, check_timelines(s, calls, speed, busy, (j, mode), oracle))]
                if j % 4 == 0:
                    ident += check_identities(s, calls)
                if j == 1 and not mode:
                    check_refusals(s, *calls[1], speed, busy)
            finally:
                s.close()
    assert tot[0] > (100 if EMULATED else 2000) and tot[1] > 0 and tot[2] > 0 and ident > 0, (tot, ident)


@pytest.mark.gpu
def test_forecast_pending_with_arrivals_on_the_gpu():
    from tests.test_plan import _gpu_factory
    assert _against_the_reference(_gpu_factory(), limit=3 if EMULATED else None) > 0


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After config 4's solve: a burst of 4 096 one-GPU arrivals at one clock in gap 1 and a spread of 4 096 over 8
    scans, with and without departures of placed pods, on the mirror and on the snapshot.  Each equals
    ``nhd_plan_scenarios_arrivals`` with the same single scenario, and 64 sampled pods' bindings equal the oracle's."""
    import workload
    from nhd_b200.solver import Solver
    from tests.test_forecast import _steps
    from tests.test_forecast_batch import config4_pending
    recs, speed, pods, now = workload.make_workload(4)
    recs, tail = config4_pending(recs, pods, 4096, 64)
    rng = np.random.default_rng(46)
    s = Solver(speed, min_busy_secs=30.0)
    try:
        s.load_nodes(recs)
        b0 = s.solve_batch(pods, now)
        after = s.read_nodes()
        s.snapshot()
        t = float(now.max()) + 5.0
        rounds = _steps(t, 30.0, 8)
        placed = np.flatnonzero(b0['status'] == wire.PLACED)
        p = tail[rng.integers(0, len(tail), 4096)]
        n_checked = 0
        for spread in (False, True):
            if spread:
                gaps = np.sort(rng.integers(1, len(rounds) + 1, len(p)))
                lo = np.where(gaps == 1, t, np.asarray([t] + list(rounds))[gaps - 1])
                clock = lo + rng.random(len(p)) * (np.asarray(rounds)[gaps - 1] - lo)
                order = np.lexsort((clock, gaps))
                arrive, clock = gaps[order].astype('<i4'), clock[order]
            else:
                arrive, clock = np.ones(len(p), dtype='<i4'), np.full(len(p), t + 1.0)
            for departures in (False, True):
                rels = np.zeros(0, dtype=wire.RELEASE_DTYPE)
                if departures:
                    rl = []
                    for q, i in enumerate(rng.choice(placed, 64, replace=False)):
                        rnd = 1 + q % len(rounds)
                        lo = t if rnd == 1 else rounds[rnd - 2]
                        rl.append(release_of(b0[i], pods[i], int(b0[i]['node']), rnd,
                                             lo + 0.5 * (rounds[rnd - 1] - lo), 1 + int(rng.integers(2))))
                    rels = np.array(sorted(rl, key=lambda x: (int(x['round']), float(x['clock']))),
                                    dtype=wire.RELEASE_DTYPE)
                tracked = sorted({int(x['node']) for x in rels})
                used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
                for q, node in enumerate(tracked):
                    nn = int(after['n_nics'][node])
                    used[q, :nn] = [int(after['nic_inuse'][node]) >> i & 1 for i in range(nn)]
                sc = Scenario((), p, clock, None, None, None, rounds, (tracked, used, rels), arrive)
                (code, _, sb, srnd, sclk), = s.plan_scenarios([sc])
                assert code == 0
                for source in ('mirror', 'snapshot'):
                    b, rnd, clk = s.plan_batch_arrivals(p, clock, rounds, tracked, used, rels, arrive, source=source)
                    assert b.tobytes() == sb.tobytes(), (spread, departures, source, helpers.first_binding_diff(sb, b))
                    assert (rnd == srnd).all() and clk.tobytes() == sclk.tobytes(), (spread, departures, source)
                    assert int((b['status'] == wire.PLACED).sum()) > 0
                if not departures:
                    k = 64
                    sub = Scenario((), p[:k], clock[:k], None, None, None, rounds, (tracked, used, rels), arrive[:k])
                    wb, wrnd, _, wclk = oracle_scenario_arrivals(after, speed, sub, busy=30.0)
                    b, rnd, clk = s.plan_batch_arrivals(p[:k], clock[:k], rounds, tracked, used, rels, arrive[:k])
                    assert b.tobytes() == wb.tobytes() and (rnd == wrnd).all() and clk.tobytes() == wclk.tobytes()
                    n_checked += k
        assert n_checked > 0
    finally:
        s.close()
