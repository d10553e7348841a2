"""Pending-queue forecasts: scenarios retried over later scans (``nhd_plan_scenarios_rounds``, ``Solver.plan_scenarios``
with rounds, ``DeviceCluster.plan_scenarios``, ``NHDScheduler.ForecastPending``).

The contract is "the five steps on a grown scratch copy, then ``nhd_solve_batch`` of the pods not placed yet at each
round's clock": scenario s gets, byte for byte, each pod's last attempt on that copy, node indices mapped back, the
round that placed each pod, and the reasons of the pods whose last attempt found no node at that attempt.  The chain
of evidence:
  * ``ForecastPending``, answered by that oracle, equals the scan that bound each pending pod and its node in the
    unmodified reference running several pending scans with its clock stepped between them, and the reference's own
    drop decisions at the last scan, frozen in tests/golden/live/forecast.json.gz (no GPU);
  * the scenario kernel, run on the CPU emulation of the device (tests/emu) in both lane orders, equals the oracle per
    scenario (bindings, rounds, reasons), also where failed assignments walk a pod across more nodes than the scenario
    has pods, refuses every malformed round argument, and without rounds is ``nhd_plan_scenarios_grown`` (no GPU);
  * on the GPU every scenario equals a scratch handle running the five steps and the round solves in every sweep mode,
    the call changes nothing of the handle's state, and so at config 4's full size (``-m gpu``)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import wire
from nhd_b200.solver import Scenario
from tests import helpers
from tests.plan_oracle import OraclePlanner, grown, mapped, oracle_scenario
from tests.test_expand import _raw as _raw_grown, expand_scenarios
from tests.test_plan import _emu_lib, _gpu_factory
from tests.test_query import MODES, _filter_words, _gpu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


# ---------------------------------------------------------------------------------------------- scenario families
def _steps(t0, period, k):
    """``k`` clocks, each the one before plus ``period`` (the way a clock advances), from ``t0``."""
    out, t = [], float(t0)
    for _ in range(k):
        t = t + period
        out.append(t)
    return out


def forecast_scenarios(recs0, pods, now, nodes_of, rest, busy):
    """The scenario families on one state: ``expand_scenarios``' families (additions, drains held to the end and
    lifted, edits, an empty scenario) each with later rounds, periods cycling through ``busy``, ``busy`` + 1, a third
    of ``busy`` and ``busy`` from a fractional start clock, 1 to 8 rounds; the plain pending tail with rounds and none
    (``rounds`` given as an empty list); a scenario whose rounds have all placed before they run."""
    tail, tclock = rest
    base = expand_scenarios(recs0, pods, now, nodes_of, rest)
    out = []
    for j, sc in enumerate(base):
        c = float(np.max(sc[2])) if len(sc[2]) else float(now[0]) if len(now) else 1000.0
        period = (busy, busy + 1.0, busy / 3.0, busy)[j % 4] or 10.0
        start = c + (0.1 if j % 4 == 3 else 0.0)
        k = 1 + j % 8
        out.append(tuple(sc) + ([start] + _steps(start, period, k - 1),))
    c = float(np.max(tclock)) if len(tclock) else 1000.0
    out.append(((), tail, tclock, None, None, None, _steps(c, busy or 10.0, 3)))
    out.append(((), tail, tclock, None, None, None, []))
    out.append(((), tail[:1], tclock[:1], None, None, None, _steps(c, 1.0, 2)))
    return out


def walker():
    """A pod whose assignment fails on more than one node, retried every 10 s (a third of the busy window) over twelve
    rounds: each failure stamps its node busy, so a later round moves it on to the next node and its scenario touches
    more nodes than it has pods.  ``(recs, pods, now, speed, busy, scenarios)``: query stream 'wild' 5, pod 25 on the
    stream's start, alone and with a second pod."""
    from tests.test_query import query_streams
    scn = dict(query_streams())['wild'][5]
    recs, pods, now, speed, busy = packed(scn)
    c = float(now.max())
    rounds = _steps(c, busy / 3.0, 12)
    scens = [((), pods[[25]], np.full(1, c), None, None, None, rounds),
             ((), pods[[25, 0]], np.full(2, c), None, None, None, rounds)]
    return recs, pods, now, speed, busy, scens


def check_against_oracle(got, scens, st, speed, busy, where='', explain=False):
    """Every scenario equals the oracle on ``st``: returns the pods compared, the pods placed at a round >= 1, and the
    most touched nodes per scenario pod seen."""
    n = later = 0
    walk = 0.0
    base = 0
    for j, (sc, g) in enumerate(zip(scens, got)):
        sc = Scenario(*sc)
        p, adds = sc.pods, sc.adds
        assert g[0] == 0 and g[1] == -1 and len(g[2]) == len(p), (where, j, g[:2])
        if len(p):
            b, rnd, rows, touched = oracle_scenario(st, speed, sc, base, busy, explain=explain)
            assert g[2].tobytes() == b.tobytes(), (where, j, helpers.first_binding_diff(b, g[2]))
            assert (g[-1] == rnd).all(), (where, j, g[-1], rnd)
            if explain:
                bad = (g[3] != rows).any(1)
                assert not bad.any(), (where, j, np.flatnonzero(bad), g[3][bad][:2], rows[bad][:2])
                none = g[2]['status'] == wire.NO_CANDIDATE
                assert (g[3][none].sum(1) == len(st) + (0 if adds is None else len(adds[0]))).all(), (where, j)
            n += len(p)
            later += int(((g[-1] >= 1) & (g[2]['status'] == wire.PLACED)).sum())
            walk = max(walk, len(touched) / len(p))
        base += 0 if adds is None else len(adds[0])
    return n, later, walk


def _raw(s, scens, round_start=True, fill=None, pod_round=True):
    """``nhd_plan_scenarios_rounds`` itself (``round_start=False``: NULL): ``(rc, status, which, out, counts,
    pod_round)``."""
    n = len(scens)
    parts = [Scenario(*sc) for sc in scens]
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), dtype=dt)  # noqa: E731
    off = lambda ls: np.concatenate([[0], np.cumsum(ls)]).astype('<i4')                           # noqa: E731
    ex = cat([np.asarray(p.exclude, dtype='<i4').reshape(-1) for p in parts], '<i4')
    pods = cat([p.pods for p in parts], wire.POD_DTYPE)
    now = cat([np.asarray(p.now, dtype='<f8') for p in parts], '<f8')
    lift = np.asarray([len(p.pods) if p.lift is None else p.lift for p in parts], dtype='<i4')
    edn = cat([np.asarray([] if p.edits is None else p.edits[0], dtype='<i4') for p in parts], '<i4')
    edr = cat([p.edits[1] for p in parts if p.edits is not None], wire.NODE_DTYPE)
    adat = cat([np.asarray([] if p.adds is None else p.adds[0], dtype='<i4') for p in parts], '<i4')
    adr = cat([p.adds[1] for p in parts if p.adds is not None], wire.NODE_DTYPE)
    clk = cat([np.asarray([] if p.rounds is None else p.rounds, dtype='<f8') for p in parts], '<f8')
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    status, which = np.zeros(n, dtype='<i4'), np.zeros(n, dtype='<i4')
    counts = None if fill is None else np.full((len(pods), wire.WHY_COUNT), fill, dtype='<u4')
    rnd = np.full(len(pods), -7, dtype='<i4') if pod_round else None
    ptr = lambda a: a.ctypes.data if a is not None and len(a) else None                           # noqa: E731
    excl_start, pod_start = off([len(p.exclude) for p in parts]), off([len(p.pods) for p in parts])
    edit_start = off([0 if p.edits is None else len(p.edits[0]) for p in parts])
    astart = off([0 if p.adds is None else len(p.adds[0]) for p in parts])
    rstart = off([0 if p.rounds is None else len(p.rounds) for p in parts])
    rc = s._L.nhd_plan_scenarios_rounds(s._h, 0, n, excl_start.ctypes.data, ptr(ex), lift.ctypes.data,
                                        edit_start.ctypes.data, ptr(edn), ptr(edr), astart.ctypes.data, ptr(adat),
                                        ptr(adr), pod_start.ctypes.data, ptr(pods), ptr(now),
                                        rstart.ctypes.data if round_start else None, ptr(clk), ptr(out),
                                        status.ctypes.data, which.ctypes.data, ptr(counts), ptr(rnd))
    return rc, status, which, out, counts, rnd


def check_refusals(s, recs, pods, now):
    """Every malformed round argument refuses the whole call; a bad pod refuses its scenario only; without rounds the
    call is ``nhd_plan_scenarios_grown`` byte for byte, ``pod_round`` all zero."""
    from nhd_b200.solver import SolverError

    def refused(scens, what):
        with pytest.raises(SolverError) as e:
            s.plan_scenarios(scens)
        assert e.value.code == wire.ERR_INVALID and what in str(e.value), str(e.value)
    t = float(np.max(now))
    refused([((), pods, now, None, None, None, [t + 1.0, float('nan')])], 'not finite')
    refused([((), pods, now, None, None, None, [float('inf')])], 'not finite')
    refused([((), pods, now, None, None, None, [t + 30.0, t + 10.0])], 'go down')
    refused([((), pods, now, None, None, None, [t - 1.0])], 'earlier than')
    refused([((), pods[:1], now[:1], None, None, None, []), ((), pods, now, None, None, None, [t - 1.0])], 'earlier than')
    L, h = s._L, s._h
    i32 = lambda *v: (ctypes.c_int32 * len(v))(*v)                           # noqa: E731
    f64 = lambda *v: (ctypes.c_double * len(v))(*v)                          # noqa: E731
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    head = (h, 0, 1, i32(0, 0), None, None, None, None, None, None, None, None, i32(0, len(pods)), pods.ctypes.data,
            now.ctypes.data)
    tail = (out.ctypes.data, i32(0), i32(0), None, None)
    assert L.nhd_plan_scenarios_rounds(*head, i32(0, 1), f64(t), *tail) == 0
    assert L.nhd_plan_scenarios_rounds(*head, i32(1, 1), f64(t), *tail) == wire.ERR_INVALID        # not from 0
    assert L.nhd_plan_scenarios_rounds(h, 0, 2, i32(0, 0, 0), None, None, None, None, None, None, None, None,
                                       i32(0, len(pods), len(pods)), pods.ctypes.data, now.ctypes.data, i32(0, 2, 1),
                                       f64(t, t), out.ctypes.data, i32(0, 0), i32(0, 0), None, None) == wire.ERR_INVALID
    assert L.nhd_plan_scenarios_rounds(*head, i32(0, 1), None, *tail) == wire.ERR_INVALID          # null clocks
    # a refused scenario in the middle: the others are planned, its pod_round rows are not written
    bad = pods.copy()
    bad[1]['n_groups'] = 0
    got = s.plan_scenarios([((), pods, now, None, None, None, [t + 30.0]), ((), bad, now, None, None, None, [t]),
                            ((), pods, now, None, None, None, [t + 30.0])])
    assert got[0][0] == 0 and got[1] == (wire.ERR_INVALID, 1, None, None) and got[2][0] == 0
    assert got[0][2].tobytes() == got[2][2].tobytes() and (got[0][3] == got[2][3]).all()
    # round_start NULL: nhd_plan_scenarios_grown byte for byte, pod_round zeroed
    one = recs[[0]].copy()
    scens = [((), pods, now, None, None, ([0], one)), ((), pods[::-1], now[::-1])]
    for fill in (None, 7):
        rc, st, wh, o, cnt, rnd = _raw(s, scens, round_start=False, fill=fill)
        rc2, st2, wh2, o2, cnt2 = _raw_grown(s, scens, fill=fill)
        assert rc == rc2 == 0 and (st == st2).all() and (wh == wh2).all() and o.tobytes() == o2.tobytes()
        assert (cnt is None) or cnt.tobytes() == cnt2.tobytes()
        assert (rnd == 0).all()
    # no rounds (every scenario's list empty) through the rounds call: the same bindings again, pod_round zero
    rc, _, _, o, _, rnd = _raw(s, [sc + (None, [])[len(sc) - 5:] if len(sc) > 5 else sc + (None, None, None, [])
                                   for sc in scens])
    assert rc == 0 and o.tobytes() == o2.tobytes() and (rnd == 0).all()


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _forecast_against_the_reference(factory):
    from tests.golden import make_live_golden
    from tests.golden.make_expand_golden import candidates
    from tests.golden.make_forecast_golden import SCANS, VARIANTS, forecast_sessions
    from tests.golden.make_plan_golden import mirror_session
    from tests.test_plan_reasons import _counted
    golden = make_live_golden.load('forecast')['sessions']
    sessions = forecast_sessions()
    assert [g['name'] for g in golden] == [name for name, _ in sessions]
    n = later = unplaced = dropped = 0
    for (name, script), want in zip(sessions, golden):
        keys = [tuple(k) for k in want['pending']]
        for period, frac in VARIANTS:
            cases = [c for c in want['cases'] if (c['period'], c['frac']) == (period, frac)]
            if not cases:
                continue
            sched, k8s, clock = mirror_session(script, factory)
            try:
                state, traffic = dict(sched.pod_state), k8s.transcript()
                before = {nd: (v.maintenance, v.busy_time, list(v.pod_info)) for nd, v in sched.nodes.items()}
                clock.t += frac
                cands = candidates(sched, cases, sched._node_cls)
                got = sched.ForecastPending(SCANS, keys=keys, period=period, additions=[c for c, _ in cands],
                                            reasons=True)
                for case, (placement, reasons), (_, grown_names) in zip(cases, got, cands):
                    assert list(placement) == keys, (name, case['label'])
                    want_p = [None if p is None else (p[0], p[1]) for p in case['placed']]
                    assert list(placement.values()) == want_p, (name, case['label'], period, frac,
                                                                list(placement.values()), want_p)
                    assert reasons == _counted(case['reasons'], grown_names), (name, case['label'], period, frac)
                    n += 1
                    later += any(v is not None and v[0] >= 1 for v in placement.values())
                    unplaced += any(v is None for v in placement.values())
                    dropped += len(reasons)
                if not cases[0]['nodes']:           # the cluster as it is: one dict, and the same without reasons
                    alone = sched.ForecastPending(SCANS, keys=keys, period=period)
                    assert alone == got[0][0], name
                assert k8s.transcript() == traffic and sched.pod_state == state, name
                assert {nd: (v.maintenance, v.busy_time, list(v.pod_info)) for nd, v in sched.nodes.items()} == before
            finally:
                sched.close()
    assert n > 100 and later > 10 and unplaced > 10 and dropped > 10, (n, later, unplaced, dropped)


def test_forecast_pending_equals_the_reference_over_later_scans():
    """Which scan binds each pending pod and where, in the reference running several pending scans with its clock
    stepped by 30, 31 and 10 s and from a fractional start clock, with and without candidate nodes added, and its drop
    decisions at the last scan for the pods no scan placed, answered by ``ForecastPending`` with the oracle standing in
    for the GPU."""
    _forecast_against_the_reference(OraclePlanner)


def test_forecast_golden_places_later_and_leaves_pods_unplaced():
    from tests.golden import make_live_golden
    cases = [c for s in make_live_golden.load('forecast')['sessions'] for c in s['cases']]
    assert sum(any(p is not None and p[0] >= 1 for p in c['placed']) for c in cases) > 0
    assert sum(any(p is None for p in c['placed']) for c in cases) > 0


def test_forecast_pending_checks_its_arguments():
    from tests.golden.make_forecast_golden import forecast_sessions
    from tests.golden.make_plan_golden import mirror_session
    name, script = forecast_sessions()[-1]
    sched, _, _ = mirror_session(script, OraclePlanner)
    try:
        with pytest.raises(ValueError):
            sched.ForecastPending(0)
        with pytest.raises(ValueError):
            sched.ForecastPending(2, additions=[[(sched._node_cls('dup', True), None),
                                                 (sched._node_cls('dup', True), None)]])
        with pytest.raises(ValueError):
            sched.ForecastPending(2, additions=[[(sched._node_cls('new', True), 'no-such-node')]])
        one = sched.ForecastPending(1)
        assert all(v is None or v[0] == 0 for v in one.values())
        assert {k: None if v is None else v[1] for k, v in one.items()} == sched.PlanExpansion([[]])[0]
    finally:
        sched.close()


def test_clocks_advance_step_by_step():
    assert _steps(1000.1, 30.0, 3) == [1000.1 + 30.0, 1000.1 + 30.0 + 30.0, 1000.1 + 30.0 + 30.0 + 30.0]


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests.test_forecast import check_against_oracle, check_refusals, forecast_scenarios, walker
from tests.test_query import emu_cases, oracle_state, packed
n = later = 0
walk = 0.0
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        s.load_nodes(recs)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        first = s.solve_batch(pods[:k], now[:k])
        source = 'mirror'
        if j %% 2:                                      # a snapshot source, with the mirror moved on since
            s.snapshot()
            s.solve_batch(pods[k:2 * k], now[k:2 * k])
            source = 'snapshot'
        clock = now[k:] if j %% 3 else np.full(len(now) - k, now[k])
        scens = forecast_scenarios(recs, pods[:k], now[:k], first['node'], (pods[k:], clock), busy)
        got = s.plan_scenarios(scens, source=source, explain=bool(j %% 2))
        a, b, c = check_against_oracle(got, scens, st, speed, busy, j, explain=bool(j %% 2))
        n, later, walk = n + a, later + b, max(walk, c)
        if j == 0:
            check_refusals(s, recs, pods, now)
    finally:
        s.close()
recs, pods, now, speed, busy, scens = walker()
s = Solver(speed, min_busy_secs=busy)
try:
    s.load_nodes(recs)
    for explain in (False, True):
        walk = max(walk, check_against_oracle(s.plan_scenarios(scens, explain=explain), scens, recs, speed, busy,
                                              'walker', explain=explain)[2])
finally:
    s.close()
print('compared', later, walk, n)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_rounds_on_the_emulated_device_equal_the_oracle(lane_order):
    """``expand_scenarios``' families with 1 to 8 rounds at periods equal to, above and below the busy window and from
    a fractional start clock; a pod whose assignment fails retried below the busy window, touching more nodes than its
    scenario has pods; mirror and snapshot sources; reasons at the last attempt; the refusals and the call without
    rounds."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    later, walk, n = res.stdout.split()[-3:]
    assert int(n) > 1000 and int(later) > 50 and float(walk) > 1.0, res.stdout


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def scratch_rounds(scratch, st, scens, which=None):
    """Each scenario (those in ``which``, by default all) on ``scratch`` loaded with its grown records: the five steps,
    then ``solve_batch`` of the pods not placed yet at each round clock, exclusions held at the last pod set again for
    the rounds; node indices mapped back.  ``{j: (bindings, pod_round)}``."""
    out, base = {}, 0
    for j, sc in enumerate(scens):
        sc = Scenario(*sc)
        ex, p, c, lift, adds, rounds = sc.exclude, sc.pods, sc.now, sc.lift, sc.adds, sc.rounds
        g, ids = grown(st, sc.edits, adds, base)
        base += 0 if adds is None else len(adds[0])
        if which is not None and j not in which:
            continue
        where = np.flatnonzero(ids < len(st))
        ex = np.unique(where[np.asarray(list(ex), dtype=np.int64)]).astype('<i4')

        def flag(on):
            cur = scratch.read_nodes()[ex]
            cur['flags'] = cur['flags'] | wire.NODE_MAINTENANCE if on else held['flags']
            scratch.update_nodes(ex, cur)
        held = g[ex].copy()
        r = g.copy()
        r['flags'][ex] |= wire.NODE_MAINTENANCE
        scratch.load_nodes(r)
        n = len(p)
        lift = n if lift is None else lift
        b = np.zeros(n, dtype=wire.BINDING_DTYPE)
        if lift:
            b[:lift] = scratch.solve_batch(p[:lift], c[:lift])
        if len(ex):
            flag(False)
        if lift < n:
            b[lift:] = scratch.solve_batch(p[lift:], c[lift:])
        rnd = np.where(b['status'] == wire.PLACED, 0, len(rounds or ())).astype('<i4')
        for k, t in enumerate(rounds or (), 1):
            idx = np.flatnonzero(b['status'] != wire.PLACED)
            if not len(idx):
                continue
            if len(ex) and lift == n:
                flag(True)
            b[idx] = scratch.solve_batch(p[idx], np.full(len(idx), t))
            if len(ex) and lift == n:
                flag(False)
            rnd[idx[b['status'][idx] == wire.PLACED]] = k
        out[j] = (mapped(b, ids), rnd)
    return out


@pytest.mark.gpu
def test_rounds_equal_a_scratch_handle_and_the_oracle_in_every_sweep_mode():
    """The query tests' case families at a state the solver itself reached partway along each stream, every family of
    ``forecast_scenarios``; with reasons and without the same bindings."""
    n = later = 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::4] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s, scratch = _solver(speed, busy, **mode), _solver(speed, busy, **mode)
            try:
                s.load_nodes(recs)
                first = s.solve_batch(pods[:k], now[:k])
                after = s.read_nodes()
                for clock in (now[k:], np.full(len(pods) - k, now[k])):
                    scens = forecast_scenarios(recs, pods[:k], now[:k], first['node'], (pods[k:], clock), busy)
                    got = s.plan_scenarios(scens, explain=True)
                    want = scratch_rounds(scratch, after, scens)
                    for i, g in enumerate(got):
                        assert g[0] == 0 and g[2].tobytes() == want[i][0].tobytes(), \
                            (j, mode, i, helpers.first_binding_diff(want[i][0], g[2]))
                        assert (g[-1] == want[i][1]).all(), (j, mode, i)
                    plain = s.plan_scenarios(scens)
                    assert all(a[2].tobytes() == b[2].tobytes() and (a[-1] == b[-1]).all() for a, b in zip(got, plain))
                    if not mode:
                        a, b, _ = check_against_oracle(got, scens, st, speed, busy, j, explain=True)
                        n, later = n + a, later + b
            finally:
                s.close()
                scratch.close()
    recs, pods, now, speed, busy, scens = walker()                 # more touched nodes than pods
    for mode in MODES:
        s, scratch = _solver(speed, busy, **mode), _solver(speed, busy, **mode)
        try:
            s.load_nodes(recs)
            got = s.plan_scenarios(scens)
            want = scratch_rounds(scratch, recs, scens)
            assert all(g[2].tobytes() == want[i][0].tobytes() and (g[-1] == want[i][1]).all() for i, g in enumerate(got))
        finally:
            s.close()
            scratch.close()
    assert check_against_oracle(got, scens, recs, speed, busy, 'walker')[2] > 1.0
    assert n > (200 if EMULATED else 2000) and later > 0, (n, later)


@pytest.mark.gpu
def test_a_rounds_call_changes_nothing_and_refuses_as_documented():
    from tests.explain_scenarios import explain_scenarios
    scn = explain_scenarios()[1]
    recs, pods, now, speed, busy = packed(scn)
    s = _solver(speed, busy)
    try:
        s.load_nodes(recs)
        s.snapshot()
        b = s.solve_batch(pods, now)
        failed = int(np.flatnonzero(b['status'] == wire.NO_CANDIDATE)[0])
        timing = s.timing()
        counters = s.debug_counters()

        def state():
            words, pt = _filter_words(s)
            return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                    s.explain_batch().tobytes(), s.explain_pod(failed).tobytes())
        before = state()
        scens = forecast_scenarios(recs, pods[::-1], now[::-1], b['node'][::-1], (pods, now), busy)
        for source in ('mirror', 'snapshot'):
            s.plan_scenarios(scens, source=source)
            s.plan_scenarios(scens[:3], source=source, explain=True)
            assert state() == before, source
            assert s.timing() == timing and (s.debug_counters() == counters).all(), source
        s.query_batch(pods[:4], now[:4], source='snapshot')                           # the snapshot is still valid
        s.restore()
        assert s.read_nodes().tobytes() == recs.tobytes()
    finally:
        s.close()
    recs, pods, now, speed, busy = packed(explain_scenarios()[0])
    s = _solver(speed, busy)
    try:
        s.load_nodes(recs)
        check_refusals(s, recs, pods, now)
    finally:
        s.close()


def config4_forecast(recs, pods, clock, n_scen, n_pods, n_add, rounds, period=30.0):
    """After config 4's solve: ``n_scen`` scenarios of ``n_add`` added copies of the first GPU node's start record
    carrying a node group no source node has (at positions spread over the node order), and a pending tail of
    ``n_pods`` one-GPU pods of the batch that request that group, so that only the added nodes take them, at most one
    per added node per scan; ``rounds`` later scans ``period`` apart."""
    n = len(recs)
    bit = next(b for b in range(64) if not (np.bitwise_or.reduce(recs['group_mask']) >> np.uint64(b)) & np.uint64(1))
    cand = recs[[int(np.flatnonzero(recs['n_gpus'] > 0)[0])]].copy()
    cand['group_mask'] = np.uint64(1) << np.uint64(bit)
    gpu = pods[(pods['n_groups'] == 1) & (pods['groups']['n_gpus'][:, 0] == 1)]
    tail = np.resize(gpu, n_pods).copy()
    tail['group_mask'] = np.uint64(1) << np.uint64(bit)
    clocks = _steps(clock, period, rounds)
    scens = []
    for k in range(n_scen):
        at = np.minimum(np.sort((k * 131 + np.arange(n_add) * 997) % (n + 1)), n).astype('<i4')
        scens.append(((), tail, np.full(len(tail), clock), None, None, (at, np.repeat(cand, n_add)), clocks))
    return scens


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """16 scenarios of 1..8 added nodes with a one-GPU pending tail only they can take, over 8 scans, equal the oracle
    loop; 4 sampled ones equal a scratch handle; the tail takes more than one scan."""
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    scratch = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        s.solve_batch(pods, now)
        after = s.read_nodes()
        scens = []
        for a in range(1, 9):
            scens += config4_forecast(recs, pods, float(now.max()) + 5.0, 2, 32, a, 8)
        got = s.plan_scenarios(scens, explain=True)
        assert max(int(g[-1][g[2]['status'] == wire.PLACED].max(initial=0)) for g in got) >= 1
        sample = [int(i) for i in np.random.default_rng(4).choice(len(scens), 4, replace=False)]
        want = scratch_rounds(scratch, after, scens, set(sample))
        for i in sample:
            assert got[i][2].tobytes() == want[i][0].tobytes(), (i, helpers.first_binding_diff(want[i][0], got[i][2]))
            assert (got[i][-1] == want[i][1]).all(), i
    finally:
        s.close()
        scratch.close()
    base = 0
    for sc, g in zip(scens, got):
        adds = Scenario(*sc).adds
        b, rnd, _, _ = oracle_scenario(after, speed, sc, base, threads=os.cpu_count() or 1)
        assert g[0] == 0 and g[2].tobytes() == b.tobytes() and (g[-1] == rnd).all(), helpers.first_binding_diff(b, g[2])
        base += len(adds[0])


@pytest.mark.gpu
def test_forecast_pending_equals_the_reference_on_the_gpu():
    _forecast_against_the_reference(_gpu_factory())
