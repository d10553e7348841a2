"""Defragmentation plans: scenarios with replaced records and exclusions that end (``nhd_plan_scenarios_edited``,
``Solver.plan_scenarios``, ``DeviceCluster.plan_scenarios``, ``NHDScheduler.PlanDefrag``).

The contract is "equal to the five steps on a scratch copy": scenario s gets, byte for byte, what ``nhd_solve_batch``
returns on a copy of the source records with its edits applied and its excluded nodes in maintenance for its pods
before the lift index, back in service (their own flags) from it on.  The chain of evidence:
  * ``PlanDefrag``, answered by that oracle, equals where the unmodified reference puts the pods of a node drained
    and put back in service, and then the pending pods, frozen in tests/golden/live/defrag.json.gz (no GPU);
  * the scenario kernel, run on the CPU emulation of the device (tests/emu) in both lane orders, equals the oracle per
    scenario (no GPU);
  * on the GPU every scenario equals the five steps on a scratch handle in every sweep mode and the oracle, the call
    changes nothing of the handle's state, and so at config 4's full size (``-m gpu``)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import wire
from tests import helpers, scenarios
from tests.golden import make_live_golden
from tests.golden.make_defrag_golden import defrag_sessions
from tests.golden.make_plan_golden import mirror_session
from nhd_b200.solver import Scenario
from tests.plan_oracle import OraclePlanner, excluded, oracle_scenario
from tests.test_plan import _emu_lib, _four_numa, _gpu_factory
from tests.test_query import MODES, _filter_words, _gpu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def defrag_scenarios(recs0, pods, now, nodes_of, rest, busy):
    """The scenario families on one state.  ``recs0``: records the edits are taken from (the stream's start: a node
    with its pods released); ``nodes_of[i]``: the node pod i of ``pods`` sits on; ``rest``: ``(pods, now)`` of the
    pending tail.  Returns ``[(exclude, pods, now, lift, edits)]``:
      every node holding pods (at most six) drained, released (its start record, busy from the drain's clock) and
      back in service for the tail, at the drain's clock + ``busy`` (the first moment it takes GPU pods) and at the
      tail's own per-pod clocks; edits only (a released node and a node given another node's record); a lift only,
      half-way through a rack; an excluded node that is not edited, after the lift; lift 0; no edits and no lift."""
    nodes_of = np.asarray(nodes_of)
    rows = lambda ns: np.flatnonzero(np.isin(nodes_of, list(ns)))         # noqa: E731
    holding = sorted(set(int(n) for n in nodes_of if n >= 0))[:6]
    tail, tclock = rest
    c0 = float(now[0]) if len(now) else 1000.0

    def released(n, clock):
        r = recs0[[n]].copy()
        r['busy_time'] = clock
        return r
    out = []
    for n in holding:
        m = rows([n])
        for tc in (np.full(len(tail), c0 + busy), tclock):
            out.append(([n], np.concatenate([pods[m], tail]), np.concatenate([np.full(len(m), c0), tc]), len(m),
                        ([n], released(n, c0))))
    if len(holding) >= 2:
        a, b = holding[0], holding[-1]
        other = recs0[[(b + 1) % len(recs0)]].copy()
        out.append(((), np.concatenate([pods, tail]), np.concatenate([now, tclock]), None,
                    ([a, b], np.concatenate([released(a, c0), other]))))
        m = rows([a, b])
        out.append(([a, b], np.concatenate([pods[m], tail]), np.concatenate([np.full(len(m), c0), tclock]), len(m),
                    ([a], released(a, c0))))
        out.append(([b, a, b], np.concatenate([pods[m], tail]), np.concatenate([np.full(len(m), c0), tclock]), 0,
                    ([b], released(b, c0))))
    rack = list(range(0, min(4, len(recs0))))
    m = rows(rack)
    out.append((rack, np.concatenate([pods[m], tail]), np.concatenate([now[m], tclock]), (len(m) + len(tail)) // 2,
                None))
    out.append((rack, pods[m], now[m], None, None))
    return out


def check_against_oracle(got, scens, st, speed, busy, where=''):
    n = 0
    for j, (sc, (code, pod, b)) in enumerate(zip(scens, got)):
        sc = Scenario(*sc)
        assert code == 0 and pod == -1 and len(b) == len(sc.pods), (where, j, code, pod)
        if len(sc.pods):
            want = oracle_scenario(st, speed, sc, busy=busy)[0]
            assert b.tobytes() == want.tobytes(), (where, j, helpers.first_binding_diff(want, b))
        n += len(sc.pods)
    return n


def check_refusals(s, recs, pods, now):
    """Per-scenario refusals as ``nhd_plan_scenarios``; every malformed edit or lift refuses the whole call; the tuple
    limits count the NUMA nodes of every edit record of the call."""
    from nhd_b200.solver import SolverError

    def refused(scens, code=wire.ERR_INVALID):
        with pytest.raises(SolverError) as e:
            s.plan_scenarios(scens)
        assert e.value.code == code, str(e.value)
        return str(e.value)
    one = recs[[1]]
    bad = pods.copy()
    bad[1]['n_groups'] = 0
    got = s.plan_scenarios([([0], pods, now, 1, ([0], one)), ([0], bad, now, 1, ([0], one))])
    assert got[0][0] == 0 and got[1][:2] == (wire.ERR_INVALID, 1) and got[1][2] is None
    assert 'outside' in refused([((), pods, now, None, ([len(recs)], one))])
    assert 'outside' in refused([((), pods, now, None, ([-1], one))])
    assert 'twice' in refused([((), pods, now, None, ([2, 2], recs[[1, 1]]))])
    s.plan_scenarios([((), pods, now, None, ([2], one)), ((), pods, now, None, ([2], one))])  # once per scenario
    broken = one.copy()
    broken['n_numa'] = 0
    assert 'nhd_validate_node' in refused([((), pods, now, None, ([0], broken))])
    assert 'lift' in refused([([0], pods, now, len(pods) + 1)])
    assert 'lift' in refused([([0], pods, now, -1)])
    s.plan_scenarios([([0], pods, now, 0), ([0], pods, now, len(pods))])
    L, h = s._L, s._h
    i32 = lambda *v: (ctypes.c_int32 * len(v))(*v)                           # noqa: E731
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    st, sp = i32(0), i32(0)
    rec = np.ascontiguousarray(one)
    tail = (i32(0, len(pods)), pods.ctypes.data, now.ctypes.data, out.ctypes.data, st, sp)
    assert L.nhd_plan_scenarios_edited(h, 0, 1, i32(0, 0), None, None, i32(0, 0), None, None, *tail) == 0
    assert L.nhd_plan_scenarios_edited(h, 0, 1, i32(0, 0), None, None, i32(1, 1), i32(0), rec.ctypes.data,
                                       *tail) == wire.ERR_INVALID                         # does not start at 0
    assert L.nhd_plan_scenarios_edited(h, 0, 2, i32(0, 0, 0), None, None, i32(0, 1, 0), i32(0), rec.ctypes.data,
                                       i32(0, 1, 2), pods.ctypes.data, now.ctypes.data, out.ctypes.data, i32(0, 0),
                                       i32(0, 0)) == wire.ERR_INVALID                     # goes down
    assert L.nhd_plan_scenarios_edited(h, 0, 1, i32(0, 0), None, None, i32(0, 1), None, rec.ctypes.data,
                                       *tail) == wire.ERR_INVALID                         # no edited nodes
    assert L.nhd_plan_scenarios_edited(h, 0, 1, i32(0, 0), None, None, i32(0, 1), i32(0), None,
                                       *tail) == wire.ERR_INVALID                         # no edit records
    # the tuple limits: 4 groups are accepted on these (at most 2-NUMA) records, and refused, naming the pod, once
    # a 4-NUMA edit record is part of the call, in any scenario of it
    assert recs['n_numa'].max() <= 2
    big = pods.copy()
    big[3]['n_groups'] = 4
    for g in range(4):
        big[3]['groups'][g] = big[3]['groups'][0]
    small = big[3]['groups']                          # four one-core groups: within the per-pod limits
    small['n_proc'], small['n_helpers'], small['n_gpus'] = 1, 0, 0
    assert s.plan_scenarios([((), big, now)])[0][0] == 0
    got = s.plan_scenarios([((), big, now), ((), pods, now, None, ([0], _four_numa(recs)[[0]]))])
    assert got[0][:2] == (wire.ERR_UNSUPPORTED, 3) and got[1][0] == 0


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _defrag_against_the_reference(factory):
    golden = make_live_golden.load('defrag')['sessions']
    sessions = defrag_sessions()
    assert [g['name'] for g in golden] == [name for name, _ in sessions]
    n = moved_only = helped = 0
    for (name, script), want in zip(sessions, golden):
        sched, k8s, _ = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()

            def objs():
                return {nd: (scenarios.node_state(v), v.maintenance, v.busy_time, list(v.pod_info))
                        for nd, v in sched.nodes.items()}
            before = objs()
            counters = (sched.failed_schedule_count, sched.pods_solved, sched.cluster.batches)
            for d in want['delays']:
                got = sched.PlanDefrag(node_groups=[[c['node']] for c in d['drains']], delay=d['delay'])
                for c in d['drains']:
                    moved, pending = got[(c['node'],)]
                    assert list(moved) == [tuple(p) for p in c['moved']], (name, c['node'])
                    assert list(moved.values()) == c['moved_to'], (name, d['delay'], c['node'], list(moved.values()))
                    n += 1
                    if any(v is None for v in c['moved_to']):
                        assert pending is None, (name, c['node'])
                        moved_only += 1
                        continue
                    assert list(pending) == [tuple(p) for p in want['pending']], (name, c['node'])
                    assert list(pending.values()) == c['pending_to'], (name, d['delay'], c['node'],
                                                                       list(pending.values()))
                    helped += any(v is not None for v in pending.values())
            default = sched.PlanDefrag()                  # every node holding pods, the next scan's pods, MIN_BUSY_SECS
            assert list(default) == [(nd,) for nd, v in sched.nodes.items() if v.pod_info], name
            first = sched.PlanDefrag(node_groups=[[c['node']] for c in want['delays'][0]['drains']])
            for g, v in first.items():
                assert default[g] == v, (name, g)
            assert k8s.transcript() == traffic and sched.pod_state == state, name
            assert objs() == before, name
            assert (sched.failed_schedule_count, sched.pods_solved, sched.cluster.batches) == counters, name
            with pytest.raises(ValueError):
                sched.PlanDefrag(node_groups=[['no-such-node']])
        finally:
            sched.close()
    assert n > 150 and moved_only > 20 and helped >= 10, (n, moved_only, helped)


def test_plan_defrag_equals_the_reference_defrag():
    """Where the reference puts a drained node's pods and then the pending pods, answered before any drain by
    ``PlanDefrag`` with the oracle standing in for the GPU."""
    _defrag_against_the_reference(OraclePlanner)


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests.test_defrag import check_against_oracle, check_refusals, defrag_scenarios
from tests.test_query import emu_cases, oracle_state, packed
n = 0
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
        scens = defrag_scenarios(recs, pods[:k], np.resize(clock, k), first['node'], (pods[k:], clock), busy)
        got = s.plan_scenarios(scens, source=source)
        n += check_against_oracle(got, scens, st, speed, busy, j)
        if j == 0:
            check_refusals(s, recs, pods, now)
    finally:
        s.close()
print('compared', n)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_defrag_scenarios_on_the_emulated_device_equal_the_oracle(lane_order):
    """Mirror and snapshot sources; edits only, a lift only, both, an edited node that is excluded, an excluded node
    that is not edited after the lift, lift 0, neither; tails at the busy window's end and at per-pod clocks; mixed
    node-group lists (the explanation stream), failed assignments (the limit cases); the refusals."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    assert int(res.stdout.split()[-1]) > 1000, res.stdout


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def five_steps(scratch, scens):
    """Each scenario as ``nhd_solve_batch`` on ``scratch`` (restored to its snapshot first): the edits, the excluded
    nodes in maintenance, the pods before the lift, the excluded nodes' flags back, the rest of the pods."""
    out = []
    for sc in scens:
        sc = Scenario(*sc)
        ex, p, c, lift, edits = sc.exclude, sc.pods, sc.now, sc.lift, sc.edits
        scratch.restore()
        if edits is not None and len(edits[0]):
            scratch.update_nodes(np.asarray(edits[0], dtype='<i4'), edits[1])
        ex = np.unique(np.asarray(list(ex), dtype='<i4'))
        lift = len(p) if lift is None else lift
        held = scratch.read_nodes()[ex] if len(ex) else None
        if len(ex):
            scratch.update_nodes(ex, excluded(held, range(len(ex))))
        b = [scratch.solve_batch(p[:lift], c[:lift])] if lift else []
        if len(ex):
            back = scratch.read_nodes()[ex]
            back['flags'] = held['flags']
            scratch.update_nodes(ex, back)
        if lift < len(p):
            b.append(scratch.solve_batch(p[lift:], c[lift:]))
        out.append(np.concatenate(b) if b else np.zeros(0, dtype=wire.BINDING_DTYPE))
    return out


def _same_as_five_steps(got, want, where=''):
    assert len(got) == len(want), where
    for j, ((code, _, b), w) in enumerate(zip(got, want)):
        assert code == 0 and b.tobytes() == w.tobytes(), (where, j, helpers.first_binding_diff(w, b))


def _plain(s, scens):
    """``nhd_plan_scenarios`` itself, for scenarios without edits or lift."""
    pods = np.concatenate([sc[1] for sc in scens]).astype(wire.POD_DTYPE)
    now = np.concatenate([np.asarray(sc[2], dtype='<f8') for sc in scens])
    ex = np.concatenate([np.asarray(sc[0], dtype='<i4').reshape(-1) for sc in scens] + [np.zeros(1, dtype='<i4')])
    excl_start = np.concatenate([[0], np.cumsum([len(sc[0]) for sc in scens])]).astype('<i4')
    pod_start = np.concatenate([[0], np.cumsum([len(sc[1]) for sc in scens])]).astype('<i4')
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    status = np.zeros(len(scens), dtype='<i4')
    which = np.zeros(len(scens), dtype='<i4')
    assert s._L.nhd_plan_scenarios(s._h, 0, len(scens), excl_start.ctypes.data, ex.ctypes.data, pod_start.ctypes.data,
                                   pods.ctypes.data, now.ctypes.data, out.ctypes.data, status.ctypes.data,
                                   which.ctypes.data) == 0
    assert (status == 0).all()
    return out


@pytest.mark.gpu
def test_defrag_scenarios_equal_the_five_steps_and_the_oracle_in_every_sweep_mode():
    """The query tests' case families at a state the solver itself reached partway along each stream; every family of
    ``defrag_scenarios``; the same scenarios without edits and lift equal ``nhd_plan_scenarios`` byte for byte."""
    n = 0
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
                scratch.load_nodes(s.read_nodes())
                scratch.snapshot()
                for clock in (now[k:], np.full(len(pods) - k, now[k])):
                    scens = defrag_scenarios(recs, pods[:k], np.resize(clock, k) if len(clock) else now[:k],
                                             first['node'], (pods[k:], clock), busy)
                    got = s.plan_scenarios(scens)
                    _same_as_five_steps(got, five_steps(scratch, scens), (j, mode))
                    bare = [tuple(sc[:3]) for sc in scens if len(sc[1])]
                    want = _plain(s, bare)
                    for form in (bare, [sc + (None, None) for sc in bare], [sc + (len(sc[1]), ([], recs[:0]))
                                                                           for sc in bare]):
                        assert np.concatenate([g[2] for g in s.plan_scenarios(form)]).tobytes() == want.tobytes()
                    if not mode:
                        n += check_against_oracle(got, scens, st, speed, busy, j)
            finally:
                s.close()
                scratch.close()
    assert n > (200 if EMULATED else 2000), n


@pytest.mark.gpu
def test_a_defrag_call_changes_nothing_and_refuses_as_documented():
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
        scens = defrag_scenarios(recs, pods[::-1], now[::-1], b['node'][::-1], (pods, now), busy)
        for source in ('mirror', 'snapshot'):
            s.plan_scenarios(scens, source=source)
            s.plan_scenarios(scens[:1], source=source)
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


def config4_defrag(pods, node, start, clock, tail):
    """After config 4's solve: one scenario per node holding pods (its pods in batch order at ``clock``, then ``tail``
    at ``clock + 30``), the node excluded until its tail and released: its record with its pods' cores, GPUs, NICs and
    hugepages back (the record before the solve), busy from ``clock``."""
    order = np.argsort(node, kind='stable')
    holding, starts = np.unique(node[order], return_index=True)
    bounds = list(starts) + [len(order)]
    out = []
    for i, n in enumerate(holding):
        if n < 0:
            continue
        m = pods[order[bounds[i]:bounds[i + 1]]]
        rec = start[[n]].copy()
        rec['busy_time'] = clock
        out.append(([int(n)], np.concatenate([m, tail]),
                    np.concatenate([np.full(len(m), clock), np.full(len(tail), clock + 30.0)]), len(m),
                    ([int(n)], rec)))
    return out


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """2 560 single-node scenarios with a pending tail (the solve's NO_CANDIDATE pods, at most 64; config 4 places every
    pod, so its first 64 pods stand in) equal the five steps on a scratch handle; 32 sampled ones equal the oracle."""
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    scratch = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        first = s.solve_batch(pods, now)
        after = s.read_nodes()
        failed = np.flatnonzero(first['status'] == wire.NO_CANDIDATE)[:64]
        tail = pods[failed] if len(failed) else pods[:64]   # config 4 places every pod: its first 64 stand in
        scens = config4_defrag(pods, first['node'], recs, float(now.max()) + 5.0, tail)
        assert len(scens) > 1000 and len(tail) > 0, (len(scens), len(tail))
        got = s.plan_scenarios(scens)
        scratch.load_nodes(after)
        scratch.snapshot()
        _same_as_five_steps(got, five_steps(scratch, scens))
        sample = [scens[i] for i in np.random.default_rng(4).choice(len(scens), 32, replace=False)]
        got = s.plan_scenarios(sample)
    finally:
        s.close()
        scratch.close()
    for sc, (code, _, b) in zip(sample, got):
        want = oracle_scenario(after, speed, sc, threads=os.cpu_count() or 1)[0]
        assert code == 0 and b.tobytes() == want.tobytes(), (sc[0], helpers.first_binding_diff(want, b))


@pytest.mark.gpu
def test_plan_defrag_equals_the_reference_defrag_on_the_gpu():
    _defrag_against_the_reference(_gpu_factory())
