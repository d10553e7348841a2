"""Forecasts of one large pending set on the batch path (``nhd_plan_batch_rounds``, ``Solver.plan_batch_rounds``,
``DeviceCluster.forecast``, ``NHDScheduler.ForecastPending`` on the cluster as it is, ``NHDScheduler.ForecastDrain``).

The contract is "``nhd_plan_batch``, then ``nhd_solve_batch`` of the pods not placed yet at each round's clock on the
records the previous round left": byte for byte each pod's last attempt, the round that placed it, and the reasons of
the pods whose last attempt found no node.  That is what ``nhd_plan_scenarios_rounds`` gives the same pods as one
scenario, so the chain of evidence is the one of tests/test_forecast.py with one more link:
  * on the CPU emulation of the device (tests/emu), both lane orders, the call equals the oracle loop
    (``plan_oracle.oracle_scenario``) and the scenario call on every family, refuses every malformed argument and moves nothing of
    the handle (no GPU);
  * ``ForecastPending`` through a solver with ``plan_batch_rounds`` equals the reference's own later scans frozen in
    tests/golden/live/forecast.json.gz and the route through the scenario call; ``ForecastDrain`` equals the oracle loop
    on the drain sessions (no GPU);
  * on the GPU the same in every sweep mode, against a scratch handle that really commits each round, and at config 4's
    full size (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import _lib, wire
from nhd_b200.solver import Scenario
from tests import helpers
from tests.plan_oracle import OraclePlanner, oracle_scenario
from tests.test_forecast import _forecast_against_the_reference, _steps, scratch_rounds, walker
from tests.test_plan import _emu_lib, _gpu_factory, exclusion_sets
from tests.test_query import MODES, _filter_words, _gpu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def test_the_symbol_is_declared_and_exported():
    from nhd_b200 import build
    build.build()
    text = open(os.path.join(ROOT, 'include', 'nhd_b200.h')).read()
    assert 'int32_t nhd_plan_batch_rounds(nhd_handle* h, int32_t source, int32_t n_excluded' in text
    assert 'nhd_plan_batch_rounds' in _lib.EXPORTS and hasattr(_lib.load(), 'nhd_plan_batch_rounds')


# ---------------------------------------------------------------------------------------------- the families
def batch_cases(recs, pods, clock, busy):
    """``(exclude, pods, now, round clocks)``: no / every third / every GPU node excluded, 1 to 8 rounds at periods of
    the busy window, one second more, a third of it, and the window from a fractional start clock; one pod (it places
    at round 0, or is retried alone); no rounds; no pods."""
    c = float(np.max(clock)) if len(clock) else 1000.0
    out = []
    for j, ex in enumerate(exclusion_sets(recs) * 2):
        period = (busy, busy + 1.0, busy / 3.0, busy)[j % 4] or 10.0
        start = c + (0.1 if j % 4 == 3 else 0.0)
        out.append((ex, pods, clock, [start] + _steps(start, period, (3 * j) % 8)))
    out.append(((), pods[:1], clock[:1], _steps(c, busy or 10.0, 3)))
    out.append((exclusion_sets(recs)[1], pods, clock, []))
    out.append(((), pods[:0], clock[:0], _steps(c, 30.0, 2)))
    return out


def check_batch_cases(s, cases, st, speed, busy, source='mirror', where=''):
    """Every case equals the oracle loop and the scenario call of the same one scenario, with reasons and without.
    Returns the pods compared, those placed at a round >= 1, and the cases where every pod of some descriptor placed at
    round 0 while other pods went on to later rounds."""
    n = later = gone = 0
    for j, (ex, p, c, rounds) in enumerate(cases):
        out, rnd, rows = s.plan_batch_rounds(p, c, rounds, source=source, exclude=ex, explain=True)
        b, wrnd, wrows, _ = oracle_scenario(st, speed, Scenario(ex, p, c, rounds=rounds), busy=busy, explain=True)
        assert out.tobytes() == b.tobytes(), (where, j, helpers.first_binding_diff(b, out))
        assert (rnd == wrnd).all(), (where, j, rnd, wrnd)
        assert (rows == wrows).all(), (where, j, np.flatnonzero((rows != wrows).any(1)))
        assert (rows[out['status'] == wire.NO_CANDIDATE].sum(1) == len(st)).all(), (where, j)
        plain, prnd = s.plan_batch_rounds(p, c, rounds, source=source, exclude=ex)
        assert plain.tobytes() == out.tobytes() and (prnd == rnd).all(), (where, j)
        if not rounds:
            one, orows = s.plan_batch(p, c, source=source, exclude=ex, explain=True)
            assert one.tobytes() == out.tobytes() and (orows == rows).all() and not rnd.any(), (where, j)
        code, _, sb, srows, srnd = s.plan_scenarios([(ex, p, c, None, None, None, rounds)], source=source,
                                                    explain=True)[0]
        if code == 0:                       # (refused only where the scenario call counts the excluded nodes' NUMA)
            assert sb.tobytes() == out.tobytes() and (srows == rows).all() and (srnd == rnd).all(), (where, j)
        else:
            assert code == wire.ERR_UNSUPPORTED and len(ex), (where, j, code)
        n += len(p)
        placed = out['status'] == wire.PLACED
        later += int((placed & (rnd >= 1)).sum())
        if len(rounds) and not placed.all():
            kinds = {}
            for i in range(len(p)):
                kinds.setdefault(p[i].tobytes(), []).append(bool(placed[i]) and rnd[i] == 0)
            gone += any(all(v) for v in kinds.values())
    return n, later, gone


def walker_cases():
    """``walker()`` as batch cases: a pod whose assignment fails on a new node at every round (each failure stamps the
    node busy), alone and followed by a pod of another descriptor that places at round 0, whose pod type then has no
    pod left in any later round."""
    recs, pods, now, speed, busy, scens = walker()
    return recs, speed, busy, [((), sc[1], sc[2], sc[6]) for sc in scens]


def check_refusals(s, recs, pods, now):
    """Every refusal of ``nhd_plan_batch_rounds`` with its code, and the NULL / zero-round forms."""
    from nhd_b200.solver import SolverError

    def refused(code, what, *args, **kw):
        with pytest.raises(SolverError) as e:
            s.plan_batch_rounds(*args, **kw)
        assert e.value.code == code and what in str(e.value), str(e.value)
    t = float(np.max(now))
    refused(wire.ERR_INVALID, 'not finite', pods, now, [t + 1.0, float('nan')])
    refused(wire.ERR_INVALID, 'not finite', pods, now, [float('inf')])
    refused(wire.ERR_INVALID, 'go down', pods, now, [t + 30.0, t + 10.0])
    refused(wire.ERR_INVALID, 'earlier than', pods, now, [t - 1.0])
    refused(wire.ERR_INVALID, f'{len(recs)}', pods, now, [t], exclude=[len(recs)])
    refused(wire.ERR_STATE, 'snapshot', pods, now, [t], source='snapshot')
    bad = pods.copy()
    bad[1]['n_groups'] = 0
    refused(wire.ERR_INVALID, 'pod 1', bad, now, [t])
    clock = now.copy()
    clock[2] = np.nan
    refused(wire.ERR_INVALID, 'pod 2', pods, clock, [t])
    L, h = s._L, s._h
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    rnd = np.full(len(pods), -7, dtype='<i4')
    clk = np.asarray([t], dtype='<f8')
    args = (len(pods), pods.ctypes.data, now.ctypes.data)
    assert L.nhd_plan_batch_rounds(h, 0, 0, None, *args, -1, clk.ctypes.data, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_rounds(h, 0, 0, None, *args, 1, None, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_rounds(h, 7, 0, None, *args, 1, clk.ctypes.data, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_rounds(h, 0, 1, None, *args, 1, clk.ctypes.data, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_rounds(h, 0, 0, None, len(pods), None, None, 1, clk.ctypes.data, None, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_rounds(None, 0, 0, None, 0, None, None, 0, None, None, None, None) == wire.ERR_INVALID
    # no rounds: nhd_plan_batch, the clocks not read, pod_round zeroed; every output but the bindings optional
    assert L.nhd_plan_batch_rounds(h, 0, 0, None, *args, 0, None, out.ctypes.data, None, rnd.ctypes.data) == 0
    assert out.tobytes() == s.plan_batch(pods, now).tobytes() and not rnd.any()
    assert L.nhd_plan_batch_rounds(h, 0, 0, None, *args, 1, clk.ctypes.data, out.ctypes.data, None, None) == 0
    assert out.tobytes() == s.plan_batch_rounds(pods, now, [t])[0].tobytes()


def check_nothing_moved(s, recs, pods, now, busy):
    """Forecasts between a solved batch and its explanations leave records, snapshot, staged batch, bindings, bitmaps,
    explanations, timing and counters as they were; the staged batch solves again to the same bindings."""
    s.load_nodes(recs)
    s.snapshot()
    b = s.solve_batch(pods, now)
    failed = int(np.flatnonzero(b['status'] == wire.NO_CANDIDATE)[0])
    timing, counters = s.timing(), s.debug_counters()

    def state():
        words, pt = _filter_words(s)
        return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                s.explain_batch().tobytes(), s.explain_pod(failed).tobytes())
    before = state()
    rounds = _steps(float(now.max()), busy / 3.0 or 10.0, 4)
    for source in ('mirror', 'snapshot'):
        for ex in exclusion_sets(recs):
            s.plan_batch_rounds(pods[::-1], np.full(len(pods), now.max()), rounds, source=source, exclude=ex, explain=True)
            s.plan_batch_rounds(pods[:1], now[:1], rounds[:1], source=source, exclude=ex)
        assert state() == before, source
        assert s.timing() == timing and (s.debug_counters() == counters).all(), source
    s.restore()
    assert s.read_nodes().tobytes() == recs.tobytes()
    s.snapshot()
    s.solve_batch(pods, now)
    s.restore()
    s.plan_batch_rounds(pods[::-1], np.full(len(pods), now.max()), rounds, exclude=exclusion_sets(recs)[1], explain=True)
    s.solve_staged()
    assert s.fetch_bindings().tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests.explain_scenarios import explain_scenarios
from tests.test_forecast_batch import (batch_cases, check_batch_cases, check_nothing_moved, check_refusals,
                                       walker_cases)
from tests.test_query import emu_cases, oracle_state, packed
n = later = gone = 0
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s, fresh = Solver(speed, min_busy_secs=busy), Solver(speed, min_busy_secs=busy)
    try:
        s.load_nodes(recs)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        s.solve_batch(pods[:k], now[:k])
        source = 'mirror'
        if j %% 2:                                      # a snapshot source, with the mirror moved on since
            s.snapshot()
            s.solve_batch(pods[k:2 * k], now[k:2 * k])
            source = 'snapshot'
        clock = now[k:] if j %% 3 else np.full(len(now) - k, now[k])
        a, b, c = check_batch_cases(s, batch_cases(recs, pods[k:], clock, busy), st, speed, busy, source, j)
        n, later, gone = n + a, later + b, gone + c
        if j == 0:
            s.load_nodes(recs)
            check_refusals(s, recs, pods, now)
        # a batch solved after forecasts equals the same batch on a fresh handle
        s.load_nodes(recs)
        fresh.load_nodes(recs)
        assert s.solve_batch(pods, now).tobytes() == fresh.solve_batch(pods, now).tobytes()
        assert s.read_nodes().tobytes() == fresh.read_nodes().tobytes()
    finally:
        s.close()
        fresh.close()
recs, speed, busy, cases = walker_cases()
s = Solver(speed, min_busy_secs=busy)
try:
    s.load_nodes(recs)
    a, b, c = check_batch_cases(s, cases, recs, speed, busy, where='walker')
    assert c >= 1, 'no pod type lost all its pods between rounds'
    out, rnd = s.plan_batch_rounds(*cases[0][1:])
    assert out['status'][0] != 0 and out['node'][0] >= 0, 'the walker no longer fails its assignment'
    recs, pods, now, speed, busy = packed(explain_scenarios()[1])
finally:
    s.close()
s = Solver(speed, min_busy_secs=busy)
try:
    check_nothing_moved(s, recs, pods, now, busy)
finally:
    s.close()
print('compared', gone + c, later, n)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_batch_rounds_on_the_emulated_device_equal_the_oracle_and_the_scenario_call(lane_order):
    """Mirror and snapshot sources; no, some and all-GPU-node exclusions; constant and per-pod clocks in round 0; mixed
    node-group lists (the explanation stream); 1 to 8 rounds at periods equal to, above and below the busy window and
    from a fractional start clock; a failed assignment retried below the busy window; pod types that lose all their
    pods between rounds; no rounds; no pods; the refusals; nothing of the handle moved."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    gone, later, n = res.stdout.split()[-3:]
    assert int(n) > 2500 and int(later) > 10 and int(gone) > 1, res.stdout


# ---------------------------------------------------------------------------------------------- CPU: the scheduler
def _without_batch_rounds(factory):
    """``factory``'s solvers with ``plan_batch_rounds`` hidden: the scheduler then takes the scenario call."""
    class Hidden:
        def __init__(self, *args, **kw):
            self._solver = factory(*args, **kw)

        def __getattr__(self, name):
            if name == 'plan_batch_rounds':
                raise AttributeError(name)
            return getattr(self._solver, name)
    return Hidden


def _routes_agree(factory, limit=None):
    """On the forecast sessions, ``ForecastPending`` of the cluster as it is through ``plan_batch_rounds`` and through
    the scenario call; on the drain sessions, ``ForecastDrain`` through ``plan_batch_rounds`` and answered by the oracle
    loop, without a Kubernetes write, and one scan of it against ``PlanDrain``."""
    from tests.golden import make_live_golden
    from tests.golden.make_forecast_golden import SCANS, VARIANTS, forecast_sessions
    from tests.golden.make_plan_golden import drain_sessions, mirror_session
    n = later = 0
    for name, script in forecast_sessions()[:limit]:
        for period, frac in VARIANTS:
            got = []
            for f in (factory, _without_batch_rounds(factory)):
                sched, _, clock = mirror_session(script, f)
                try:
                    clock.t += frac
                    got.append(sched.ForecastPending(SCANS, period=period, reasons=True))
                finally:
                    sched.close()
            assert got[0] == got[1], (name, period, frac)
            n += len(got[0][0])
            later += sum(v is not None and v[0] >= 1 for v in got[0][0].values())
    assert limit is not None or (n > 20 and later > 0), (n, later)
    n = later = 0
    golden = make_live_golden.load('plan')['sessions']
    for (name, script, _), want in list(zip(drain_sessions(), golden))[:limit]:
        got = []
        for f in (factory, OraclePlanner):
            sched, k8s, _ = mirror_session(script, f)
            try:
                state, traffic = dict(sched.pod_state), k8s.transcript()
                got.append([sched.ForecastDrain(want['drain'], 4, period=p, reasons=True) for p in (None, 10.0)])
                assert k8s.transcript() == traffic and sched.pod_state == state, name
                if f is factory:
                    placement, why = sched.PlanDrain(want['drain'])
                    one = sched.ForecastDrain(want['drain'], 1, reasons=True)
                    assert one == ({k: None if v is None else (0, v) for k, v in placement.items()}, why), name
                    assert sched.ForecastDrain(want['drain'], 1) == one[0]
                    with pytest.raises(ValueError):
                        sched.ForecastDrain(['no-such-node'], 2)
                    with pytest.raises(ValueError):
                        sched.ForecastDrain(want['drain'], 0)
            finally:
                sched.close()
        assert got[0] == got[1], name
        assert list(got[0][0][0]) == [tuple(p) for p in want['pods']], name
        n += len(got[0][0][0])
        later += sum(v is not None and v[0] >= 1 for v in got[0][0][0].values())
    assert limit is not None or (n > 20 and later > 0), (n, later)


SCHED_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
from tests.test_forecast import _forecast_against_the_reference
from tests.test_forecast_batch import _routes_agree
from tests.test_plan import _gpu_factory
_forecast_against_the_reference(_gpu_factory())
_routes_agree(_gpu_factory(), limit=4)
print('ok')
'''


def test_the_scheduler_on_the_emulated_device_equals_the_reference_on_both_routes():
    """``ForecastPending`` with the emulated device behind the scheduler (a solver with ``plan_batch_rounds``) equals
    the reference's later scans in tests/golden/live/forecast.json.gz, and the route through the scenario call;
    ``ForecastDrain`` equals the oracle loop, writes nothing, and with one scan is ``PlanDrain``."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d')
    res = subprocess.run([sys.executable, '-c', SCHED_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0 and res.stdout.split()[-1] == 'ok', (res.stdout + res.stderr)[-3000:]


def test_forecast_drain_with_the_oracle_stand_in_takes_the_scenario_call():
    """A solver without ``plan_batch_rounds``: ``ForecastDrain`` through the scenario call, one scan of it ``PlanDrain``."""
    from tests.golden import make_live_golden
    from tests.golden.make_plan_golden import drain_sessions, mirror_session
    (name, script, _), want = drain_sessions()[0], make_live_golden.load('plan')['sessions'][0]
    sched, _, _ = mirror_session(script, OraclePlanner)
    try:
        placement, why = sched.PlanDrain(want['drain'])
        assert sched.ForecastDrain(want['drain'], 1, reasons=True) == \
            ({k: None if v is None else (0, v) for k, v in placement.items()}, why)
        more = sched.ForecastDrain(want['drain'], 4)
        assert all(more[k] == (0, v) for k, v in placement.items() if v is not None)
    finally:
        sched.close()


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


@pytest.mark.gpu
def test_batch_rounds_equal_the_oracle_the_scenario_call_and_a_scratch_handle_in_every_sweep_mode():
    """The query tests' case families at a state the solver itself reached partway along each stream; every family of
    ``batch_cases`` against the oracle loop and the scenario call, and against a scratch handle that really does it
    (load, maintenance, per round: solve the unplaced pods); the walker in every mode."""
    n = later = gone = 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::6] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s, scratch = _solver(speed, busy, **mode), _solver(speed, busy, **mode)
            try:
                s.load_nodes(recs)
                s.solve_batch(pods[:k], now[:k])
                after = s.read_nodes()
                for clock in (now[k:], np.full(len(pods) - k, now[k])):
                    bc = batch_cases(recs, pods[k:], clock, busy)
                    a, b, c = check_batch_cases(s, bc, st, speed, busy, where=(j, mode))
                    n, later, gone = n + a, later + b, gone + c
                    want = scratch_rounds(scratch, after, [(ex, p, c_, None, None, None, r) for ex, p, c_, r in bc[:-1]])
                    for i, (ex, p, c_, r) in enumerate(bc[:-1]):
                        out, rnd = s.plan_batch_rounds(p, c_, r, exclude=ex)
                        assert out.tobytes() == want[i][0].tobytes() and (rnd == want[i][1]).all(), (j, mode, i)
            finally:
                s.close()
                scratch.close()
    recs, speed, busy, wc = walker_cases()
    for mode in MODES:
        s = _solver(speed, busy, **mode)
        try:
            s.load_nodes(recs)
            assert check_batch_cases(s, wc, recs, speed, busy, where=('walker', mode))[2] >= 1
        finally:
            s.close()
    assert n > (100 if EMULATED else 2000) and later > 0 and gone > 0, (n, later, gone)


@pytest.mark.gpu
def test_a_batch_forecast_changes_nothing_and_refuses_as_documented():
    from tests.explain_scenarios import explain_scenarios
    recs, pods, now, speed, busy = packed(explain_scenarios()[1])
    s = _solver(speed, busy)
    try:
        check_nothing_moved(s, recs, pods, now, busy)
    finally:
        s.close()
    recs, pods, now, speed, busy = packed(explain_scenarios()[0])
    s, fresh = _solver(speed, busy), _solver(speed, busy)
    try:
        from nhd_b200.solver import SolverError
        with pytest.raises(SolverError) as e:
            s.plan_batch_rounds(pods, now, [float(now.max())])
        assert e.value.code == wire.ERR_STATE                                  # nothing loaded
        s.load_nodes(recs)
        fresh.load_nodes(recs)
        check_refusals(s, recs, pods, now)
        assert s.solve_batch(pods, now).tobytes() == fresh.solve_batch(pods, now).tobytes()
        assert s.read_nodes().tobytes() == fresh.read_nodes().tobytes()
    finally:
        s.close()
        fresh.close()


def config4_pending(recs, pods, n_pods, n_nodes):
    """Config 4 with a node group only ``n_nodes`` of its GPU nodes carry (besides their own), and ``n_pods`` one-GPU
    pods of the stream that request it: each scan places at most one per such node, the rest find no node."""
    bit = next(b for b in range(64) if not (np.bitwise_or.reduce(recs['group_mask']) >> np.uint64(b)) & np.uint64(1))
    recs = recs.copy()
    gpu_nodes = np.flatnonzero(recs['n_gpus'] > 0)
    recs['group_mask'][gpu_nodes[::max(1, len(gpu_nodes) // n_nodes)][:n_nodes]] |= np.uint64(1) << np.uint64(bit)
    gpu = pods[(pods['n_groups'] == 1) & (pods['groups']['n_gpus'][:, 0] == 1)]
    tail = np.resize(gpu, n_pods).copy()
    tail['group_mask'] = np.uint64(1) << np.uint64(bit)
    return recs, tail


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After config 4's solve, a pending set of 4 096 pods over 8 scans equals ``nhd_plan_scenarios_rounds`` of the same
    one scenario on every field, with and without 1 024 exclusions; 32 sampled pods, forecast as a pending set of their
    own from the same state, equal the oracle loop."""
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    recs, tail = config4_pending(recs, pods, 4096, 64)
    s = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        s.solve_batch(pods, now)
        after = s.read_nodes()
        t = float(now.max()) + 5.0
        clock, rounds = np.full(len(tail), t), _steps(t, 30.0, 8)
        for ex in ((), tuple(range(7, len(recs), 64))[:1024]):
            out, rnd, rows = s.plan_batch_rounds(tail, clock, rounds, exclude=ex, explain=True)
            code, _, sb, srows, srnd = s.plan_scenarios([(ex, tail, clock, None, None, None, rounds)], explain=True)[0]
            assert code == 0 and sb.tobytes() == out.tobytes() and (srows == rows).all() and (srnd == rnd).all(), len(ex)
            placed = out['status'] == wire.PLACED
            assert placed.any() and not placed.all() and rnd[placed].max() >= 2, len(ex)
            assert (rows[out['status'] == wire.NO_CANDIDATE].sum(1) == len(recs)).all()
    finally:
        s.close()
    # the oracle loop on a sample: the 32 pods are the whole pending set of a cluster where they are alone in their
    # group, so the sample is planned as its own batch
    sample = np.sort(np.random.default_rng(4).choice(len(tail), 32, replace=False))
    s = _solver(speed, 30.0)
    try:
        s.load_nodes(after)
        out, rnd, rows = s.plan_batch_rounds(tail[sample], clock[sample], rounds, explain=True)
    finally:
        s.close()
    b, wrnd, wrows, _ = oracle_scenario(after, speed, Scenario((), tail[sample], clock[sample], rounds=rounds),
                                        threads=os.cpu_count() or 1, explain=True)
    assert out.tobytes() == b.tobytes() and (rnd == wrnd).all() and (rows == wrows).all(), \
        helpers.first_binding_diff(b, out)


@pytest.mark.gpu
def test_forecast_pending_and_drain_on_the_gpu():
    if not EMULATED:        # (on the emulated device the CPU suite already runs this, in a process of its own)
        _forecast_against_the_reference(_gpu_factory())
    _routes_agree(_gpu_factory(), limit=1 if EMULATED else None)
