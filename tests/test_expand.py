"""Cluster growth plans: scenarios with added nodes (``nhd_plan_scenarios_grown``, ``Solver.plan_scenarios``,
``DeviceCluster.plan_scenarios``, ``NHDScheduler.PlanExpansion``).

The contract is "equal to the five steps on a grown scratch copy": scenario s gets, byte for byte, what
``nhd_solve_batch`` returns on a copy of the source records with its edits applied and its added records inserted at
their positions, its excluded nodes in maintenance for its pods before the lift index, every node index mapped back (a
source node to its index, added node a to n_nodes + a).  The chain of evidence:
  * ``PlanExpansion``, answered by that oracle, equals where the unmodified reference puts the pending pods with the
    candidate nodes inserted into its node dict, and its own drop decisions, frozen in
    tests/golden/live/expand.json.gz (no GPU);
  * the scenario kernel, run on the CPU emulation of the device (tests/emu) in both lane orders, equals the oracle per
    scenario, bindings and reasons, and refuses every malformed addition (no GPU);
  * on the GPU every scenario equals the five steps on a scratch handle loaded with the grown records in every sweep
    mode and the oracle, the call changes nothing of the handle's state, and so at config 4's full size (``-m gpu``)."""
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
from tests.test_plan import _emu_lib, _gpu_factory
from tests.test_query import MODES, _filter_words, _gpu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


# ---------------------------------------------------------------------------------------------- scenario families
def _shapes(recs0):
    """Up to three distinct node shapes of ``recs0`` (the stream's start: nodes without pods): indices."""
    seen, out = set(), []
    for i in range(len(recs0)):
        key = (int(recs0['n_gpus'][i]), int(recs0['n_numa'][i]), int(recs0['phys_cores'][i]), int(recs0['n_nics'][i]))
        if key not in seen:
            seen.add(key)
            out.append(i)
    return out[:3]


def expand_scenarios(recs0, pods, now, nodes_of, rest):
    """The scenario families on one state.  ``recs0``: records the added nodes are taken from (the stream's start);
    ``nodes_of[i]``: the node pod i of ``pods`` sits on; ``rest``: ``(pods, now)`` of the pending tail.  Returns
    ``[(exclude, pods, now, lift, edits, adds)]``: one copy of each shape at the end, the front and the middle; 1, 2
    and 3 copies at one position; several positions in one scenario; a GPU-less node; another NUMA count; a node in
    maintenance and an inactive one; a node-group set no node has; a drained node replaced by an added one (exclusion
    held, and lifted with the node released); additions with edits; an empty scenario."""
    n = len(recs0)
    tail, tclock = rest
    nodes_of = np.asarray(nodes_of)
    out = []

    def add(at, idx, tweak=None):
        r = recs0[np.asarray(idx, dtype=np.int64)].copy()
        if tweak is not None:
            tweak(r)
        return (np.asarray(at, dtype='<i4'), r)
    shapes = _shapes(recs0)
    for i in shapes:
        for at in (n, 0, n // 2):
            out.append(((), tail, tclock, None, None, add([at], [i])))
    s0 = shapes[0]
    for k in (1, 2, 3):
        out.append(((), tail, tclock, None, None, add([n // 2] * k, [s0] * k)))
    out.append(((), tail, tclock, None, None, add([0, n // 3, n // 3, n], shapes[:1] * 2 + shapes[-1:] * 2)))

    def gpuless(r):
        r['n_gpus'] = 0
        r['gpu_used'] = 0
        r['gpu_numa_mask'] = 0
        r['gpu_sw'] = 0
    out.append(((), tail, tclock, None, None, add([0], [s0], gpuless)))
    other = [i for i in range(n) if recs0['n_numa'][i] != recs0['n_numa'][s0]]
    if other:
        out.append(((), tail, tclock, None, None, add([0, n], [other[0], s0])))
    out.append(((), tail, tclock, None, None, add([0], [s0], lambda r: r.__setitem__('flags', r['flags'] | wire.NODE_MAINTENANCE))))
    out.append(((), tail, tclock, None, None, add([0], [s0], lambda r: r.__setitem__('flags', r['flags'] & (0xFF ^ wire.NODE_ACTIVE)))))
    masks = set(int(m) for m in recs0['group_mask'])
    fresh = next(1 << b for b in range(64) if not any(m & (1 << b) for m in masks))
    for m in sorted(masks)[:2]:
        out.append(((), tail, tclock, None, None, add([n // 2, n], [s0, s0],
                                                      lambda r, m=m: r.__setitem__('group_mask', [m ^ fresh, m]))))
    holding = sorted(set(int(x) for x in nodes_of if x >= 0))[:3]
    for h in holding:
        moved = np.flatnonzero(nodes_of == h)
        rel = recs0[[h]].copy()
        out.append(([h], np.concatenate([pods[moved], tail]), np.concatenate([now[moved], tclock]), None, None,
                    add([h], [h])))
        out.append(([h], np.concatenate([pods[moved], tail]), np.concatenate([now[moved], tclock]), len(moved),
                    ([h], rel), add([h, n], [h, s0])))
    if len(holding) >= 2:
        out.append(((), tail, tclock, None, ([holding[0]], recs0[[holding[0]]]), add([holding[1]], [s0])))
    out.append(((), tail[:0], tclock[:0], None, None, add([0], [s0])))
    return out


def check_against_oracle(got, scens, st, speed, busy, where='', explain=False, refused=()):
    """Every accepted scenario equals the oracle on ``st``, added nodes numbered call-wide; returns the pods compared
    and the pods placed on added nodes."""
    n = on_added = base = 0
    for j, (sc, g) in enumerate(zip(scens, got)):
        sc = Scenario(*sc)
        adds = sc.adds
        if j in refused:
            assert g[0] == refused[j][0] and g[1] == refused[j][1] and g[2] is None, (where, j, g[:2])
        else:
            assert g[0] == 0 and g[1] == -1 and len(g[2]) == len(sc.pods), (where, j, g[:2])
            if len(sc.pods):
                b, _, rows, _ = oracle_scenario(st, speed, sc, base, busy, explain=explain)
                assert g[2].tobytes() == b.tobytes(), (where, j, helpers.first_binding_diff(b, g[2]))
                if explain:
                    bad = (g[3] != rows).any(1)
                    assert not bad.any(), (where, j, np.flatnonzero(bad), g[3][bad][:2], rows[bad][:2])
                    none = g[2]['status'] == wire.NO_CANDIDATE
                    assert (g[3][none].sum(1) == len(st) + (0 if adds is None else len(adds[0]))).all(), (where, j)
            n += len(sc.pods)
            on_added += int((g[2]['node'] >= len(st)).sum())
        base += 0 if adds is None else len(adds[0])
    return n, on_added


def _raw(s, scens, add_start=True, fill=None):
    """``nhd_plan_scenarios_grown`` itself (``add_start=False``: NULL), with a per-scenario list of ``(exclude, pods,
    now, lift, edits, adds)``: ``(rc, status, which, out, counts)``."""
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
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    status, which = np.zeros(n, dtype='<i4'), np.zeros(n, dtype='<i4')
    counts = None if fill is None else np.full((len(pods), wire.WHY_COUNT), fill, dtype='<u4')
    ptr = lambda a: a.ctypes.data if a is not None and len(a) else None                           # noqa: E731
    excl_start, pod_start = off([len(p.exclude) for p in parts]), off([len(p.pods) for p in parts])
    edit_start = off([0 if p.edits is None else len(p.edits[0]) for p in parts])
    astart = off([0 if p.adds is None else len(p.adds[0]) for p in parts])
    rc = s._L.nhd_plan_scenarios_grown(s._h, 0, n, excl_start.ctypes.data, ptr(ex), lift.ctypes.data,
                                       edit_start.ctypes.data, ptr(edn), ptr(edr),
                                       astart.ctypes.data if add_start else None, ptr(adat), ptr(adr),
                                       pod_start.ctypes.data, ptr(pods), ptr(now), ptr(out), status.ctypes.data,
                                       which.ctypes.data, ptr(counts))
    return rc, status, which, out, counts


def check_refusals(s, recs, pods, now):
    """Every malformed addition refuses the whole call; a bad pod refuses its scenario only, the added nodes of the
    others keeping their call-wide numbers; the tuple limits count the NUMA nodes of every added record."""
    from nhd_b200.solver import SolverError

    def refused(scens, what, code=wire.ERR_INVALID):
        with pytest.raises(SolverError) as e:
            s.plan_scenarios(scens)
        assert e.value.code == code and what in str(e.value), str(e.value)
    n = len(recs)
    one = recs[[0]].copy()
    refused([((), pods, now, None, None, ([-1], one))], 'outside')
    refused([((), pods, now, None, None, ([n + 1], one))], 'outside')
    refused([((), pods, now, None, None, ([2, 1], recs[[0, 0]]))], 'go down')
    broken = one.copy()
    broken['n_numa'] = 0
    refused([((), pods, now, None, None, ([0], broken))], 'nhd_validate_node')
    with_nic = recs[recs['n_nics'] > 0][:1].copy()
    assert len(with_nic)
    with_nic['nic_speed'][0, 0] = (int(with_nic['nic_speed'][0, 0]) & ~0xF) | 0xF
    refused([((), pods, now, None, None, ([0], with_nic))], 'speed class')
    # raw arguments: add offsets that do not start at 0 or go down, null added arrays
    sc = ((), pods, now, None, None, ([0], one))
    assert _raw(s, [sc])[0] == 0
    L, h = s._L, s._h
    i32 = lambda *v: (ctypes.c_int32 * len(v))(*v)                           # noqa: E731
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    rec = np.ascontiguousarray(recs[[0, 0]])
    head = (h, 0, 1, i32(0, 0), None, None, None, None, None)
    tail = (i32(0, len(pods)), pods.ctypes.data, now.ctypes.data, out.ctypes.data, i32(0), i32(0), None)
    assert L.nhd_plan_scenarios_grown(*head, i32(0, 1), i32(0), rec.ctypes.data, *tail) == 0
    assert L.nhd_plan_scenarios_grown(*head, i32(1, 1), i32(0), rec.ctypes.data, *tail) == wire.ERR_INVALID
    assert L.nhd_plan_scenarios_grown(h, 0, 2, i32(0, 0, 0), None, None, None, None, None, i32(0, 2, 1), i32(0, 0),
                                      rec.ctypes.data, i32(0, len(pods), len(pods)), pods.ctypes.data,
                                      now.ctypes.data, out.ctypes.data, i32(0, 0), i32(0, 0), None) == wire.ERR_INVALID
    assert L.nhd_plan_scenarios_grown(*head, i32(0, 1), None, rec.ctypes.data, *tail) == wire.ERR_INVALID
    assert L.nhd_plan_scenarios_grown(*head, i32(0, 1), i32(0), None, *tail) == wire.ERR_INVALID
    # a refused scenario in the middle: the last scenario's added node is still n + 2
    bad = pods.copy()
    bad[1]['n_groups'] = 0
    got = s.plan_scenarios([((), pods, now, None, None, ([0], one)), ((), bad, now, None, None, ([0], one)),
                            ((), pods, now, None, None, ([0], one))])
    assert got[0][0] == 0 and got[1][:3] == (wire.ERR_INVALID, 1, None) and got[2][0] == 0
    b0, b2 = got[0][2], got[2][2]
    assert (b0['node'] == n).any() and ((b0['node'] == n) == (b2['node'] == n + 2)).all()
    assert b0[b0['node'] != n].tobytes() == b2[b2['node'] != n + 2].tobytes()
    # the tuple limits: four one-core groups are accepted on at most 2-NUMA records, refused once a 4-NUMA added
    # record is part of the call
    if recs['n_numa'].max() <= 2:
        big = pods.copy()
        big[3]['n_groups'] = 4
        for g in range(4):
            big[3]['groups'][g] = big[3]['groups'][0]
        small = big[3]['groups']
        small['n_proc'], small['n_helpers'], small['n_gpus'] = 1, 0, 0
        assert s.plan_scenarios([((), big, now)])[0][0] == 0
        from tests.test_plan import _four_numa
        got = s.plan_scenarios([((), big, now), ((), pods, now, None, None, ([n], _four_numa(recs)[[0]]))])
        assert got[0][:2] == (wire.ERR_UNSUPPORTED, 3) and got[1][0] == 0


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _expand_against_the_reference(factory):
    from tests.golden import make_live_golden
    from tests.golden.make_expand_golden import candidates, expand_sessions
    from tests.golden.make_plan_golden import mirror_session
    from tests.test_plan_reasons import _counted
    golden = make_live_golden.load('expand')['sessions']
    sessions = expand_sessions()
    assert [g['name'] for g in golden] == [name for name, _ in sessions]
    n = helped = dropped = 0
    for (name, script), want in zip(sessions, golden):
        sched, k8s, _ = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()
            names = list(sched.nodes)
            before = {nd: (v.maintenance, v.busy_time, list(v.pod_info)) for nd, v in sched.nodes.items()}
            keys = [tuple(k) for k in want['pending']]
            cands = candidates(sched, want['cases'], sched._node_cls)
            got = sched.PlanExpansion([c for c, _ in cands], keys=keys, reasons=True)
            for case, (placement, reasons), (_, grown_names) in zip(want['cases'], got, cands):
                assert list(placement) == keys, (name, case['label'])
                assert list(placement.values()) == case['placed'], (name, case['label'], list(placement.values()))
                assert reasons == _counted(case['reasons'], grown_names), (name, case['label'])
                n += 1
                helped += any(v is not None and v not in names for v in placement.values())
                dropped += len(reasons)
            plain = sched.PlanExpansion([c for c, _ in cands], keys=keys)
            assert plain == [p for p, _ in got], name
            # additions listed out of position order land where they are inserted, named as given
            single = [c for c, _ in cands if len(c) == 1]
            other = next((c for c in single if c[0][0].name != single[0][0][0].name), None) if single else None
            both = [single[0], other] if other is not None else []
            if both:
                a, b = (both[0][0][0], None), (both[1][0][0], names[0])
                assert sched.PlanExpansion([[a, b]], keys=keys) == sched.PlanExpansion([[b, a]], keys=keys), name
            assert k8s.transcript() == traffic and sched.pod_state == state, name
            assert {nd: (v.maintenance, v.busy_time, list(v.pod_info)) for nd, v in sched.nodes.items()} == before
            with pytest.raises(ValueError):
                sched.PlanExpansion([[(sched._node_cls('dup', True), None), (sched._node_cls('dup', True), None)]],
                                    keys=keys)
            with pytest.raises(ValueError):
                sched.PlanExpansion([[(sched._node_cls('new', True), 'no-such-node')]], keys=keys)
            with pytest.raises(ValueError):
                sched.PlanExpansion([[(sched.nodes[names[0]], None)]], keys=keys)
        finally:
            sched.close()
    assert n > 100 and helped > 20 and dropped > 20, (n, helped, dropped)


def test_plan_expansion_equals_the_reference_with_the_nodes_added():
    """Where the reference puts the pending pods with candidate nodes inserted into its node dict, and its drop
    decisions for those left without a node, answered by ``PlanExpansion`` with the oracle standing in for the GPU."""
    _expand_against_the_reference(OraclePlanner)


def test_grown_records_put_added_nodes_in_front_of_their_position():
    recs = np.zeros(3, dtype=wire.NODE_DTYPE)
    recs['free_hugepages_gb'] = [10, 11, 12]
    adds = np.zeros(4, dtype=wire.NODE_DTYPE)
    adds['free_hugepages_gb'] = [20, 21, 22, 23]
    g, ids = grown(recs, None, (np.asarray([0, 2, 2, 3]), adds), base=5)
    assert ids.tolist() == [8, 0, 1, 9, 10, 2, 11]
    assert g['free_hugepages_gb'].tolist() == [20, 10, 11, 21, 22, 12, 23]


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests.test_expand import check_against_oracle, check_refusals, expand_scenarios
from tests.test_query import emu_cases, oracle_state, packed
n = on = 0
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
        scens = expand_scenarios(recs, pods[:k], now[:k], first['node'], (pods[k:], clock))
        got = s.plan_scenarios(scens, source=source, explain=bool(j %% 2))
        a, b = check_against_oracle(got, scens, st, speed, busy, j, explain=bool(j %% 2))
        n, on = n + a, on + b
        if j == 0:
            check_refusals(s, recs, pods, now)
    finally:
        s.close()
print('compared', on, n)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_grown_scenarios_on_the_emulated_device_equal_the_oracle(lane_order):
    """Additions at the end, the front, between nodes and several at one position; with edits, exclusions and a lift;
    an empty scenario; mirror and snapshot sources; constant and per-pod clocks; mixed node-group lists (the
    explanation stream); failed assignments (the limit cases); reasons against the explanation oracle on the grown
    records; the refusals."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    on, n = (int(x) for x in res.stdout.split()[-2:])
    assert n > 1000 and on > 100, res.stdout


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def five_steps_grown(scratch, st, scens, which=None):
    """Each scenario (those in ``which``, by default all) as ``nhd_solve_batch`` on ``scratch`` loaded with its grown
    records: the excluded nodes in maintenance, the pods before the lift, the excluded nodes' flags back, the rest;
    node indices mapped back."""
    out, base = {}, 0
    for j, sc in enumerate(scens):
        sc = Scenario(*sc)
        ex, p, c, lift, adds = sc.exclude, sc.pods, sc.now, sc.lift, sc.adds
        g, ids = grown(st, sc.edits, adds, base)
        base += 0 if adds is None else len(adds[0])
        if which is not None and j not in which:
            continue
        where = np.flatnonzero(ids < len(st))
        ex = np.unique(where[np.asarray(list(ex), dtype=np.int64)]).astype('<i4')
        held = g[ex].copy()
        r = g.copy()
        r['flags'][ex] |= wire.NODE_MAINTENANCE
        scratch.load_nodes(r)
        lift = len(p) if lift is None else lift
        b = [scratch.solve_batch(p[:lift], c[:lift])] if lift else []
        if len(ex):
            back = scratch.read_nodes()[ex]
            back['flags'] = held['flags']
            scratch.update_nodes(ex, back)
        if lift < len(p):
            b.append(scratch.solve_batch(p[lift:], c[lift:]))
        out[j] = mapped(np.concatenate(b), ids) if b else np.zeros(0, dtype=wire.BINDING_DTYPE)
    return [out[j] for j in sorted(out)] if which is None else out


@pytest.mark.gpu
def test_grown_scenarios_equal_the_five_steps_and_the_oracle_in_every_sweep_mode():
    """The query tests' case families at a state the solver itself reached partway along each stream; every family of
    ``expand_scenarios``; with no additions the call is ``nhd_plan_scenarios_explained`` byte for byte."""
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
                after = s.read_nodes()
                for clock in (now[k:], np.full(len(pods) - k, now[k])):
                    scens = expand_scenarios(recs, pods[:k], now[:k], first['node'], (pods[k:], clock))
                    got = s.plan_scenarios(scens, explain=True)
                    for sc, g, w in zip(scens, got, five_steps_grown(scratch, after, scens)):
                        assert g[0] == 0 and g[2].tobytes() == w.tobytes(), (j, mode, helpers.first_binding_diff(w, g[2]))
                    plain = s.plan_scenarios(scens)
                    assert all(a[2].tobytes() == b[2].tobytes() for a, b in zip(got, plain))
                    if not mode:
                        n += check_against_oracle(got, scens, st, speed, busy, j, explain=True)[0]
                    bare = [tuple(sc[:5]) for sc in scens]
                    want = s.plan_scenarios(bare, explain=True)
                    for form in (_raw(s, bare, fill=0), _raw(s, bare, add_start=False, fill=0)):
                        rc, status, _, out, counts = form
                        assert rc == 0 and (status == 0).all()
                        assert out.tobytes() == np.concatenate([w[2] for w in want]).tobytes()
                        assert counts.tobytes() == np.concatenate([w[3] for w in want]).tobytes()
            finally:
                s.close()
                scratch.close()
    assert n > (200 if EMULATED else 2000), n


@pytest.mark.gpu
def test_a_grown_call_changes_nothing_and_refuses_as_documented():
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
        scens = expand_scenarios(recs, pods[::-1], now[::-1], b['node'][::-1], (pods, now))
        for source in ('mirror', 'snapshot'):
            s.plan_scenarios(scens, source=source)
            s.plan_scenarios(scens[:1], source=source, explain=True)
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


@pytest.mark.gpu
def test_a_batch_after_grown_calls_equals_one_on_a_fresh_handle():
    for scn in _gpu_cases()[2::5][:2 if EMULATED else None]:
        recs, pods, now, speed, busy = packed(scn)
        k = len(pods) // 2
        s, fresh = _solver(speed, busy), _solver(speed, busy)
        try:
            s.load_nodes(recs)
            first = s.solve_batch(pods[:k], now[:k])
            scens = expand_scenarios(recs, pods[:k], now[:k], first['node'], (pods[k:], now[k:]))
            s.plan_scenarios(scens)
            s.plan_scenarios(scens, explain=True)
            fresh.load_nodes(s.read_nodes())
            assert s.solve_batch(pods[k:], now[k:]).tobytes() == fresh.solve_batch(pods[k:], now[k:]).tobytes()
        finally:
            s.close()
            fresh.close()


def config4_expansion(recs, pods, clock):
    """After config 4's solve: 64 scenarios of 1..64 added nodes, copies of node 0's start record carrying a node
    group no source node has, spread over the node order (scenario k: k + 1 nodes at positions k * n / 64 + i), and a
    pending tail of 64 of the batch's pods that request that group, so that only the added nodes can take them."""
    n = len(recs)
    bit = next(b for b in range(64) if not (np.bitwise_or.reduce(recs['group_mask']) >> np.uint64(b)) & np.uint64(1))
    cand = recs[[0]].copy()
    cand['group_mask'] = np.uint64(1) << np.uint64(bit)
    tail = pods[:64].copy()
    tail['group_mask'] = np.uint64(1) << np.uint64(bit)
    scens = []
    for k in range(64):
        at = np.minimum(np.sort((k * n // 64 + np.arange(k + 1) * 997) % (n + 1)), n).astype('<i4')
        scens.append(((), tail, np.full(len(tail), clock), None, None, (at, np.repeat(cand, k + 1))))
    return scens


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """64 scenarios of 1..64 added nodes with a pending tail only they can take equal the oracle; 8 sampled ones
    equal the five steps on a scratch handle loaded with the grown records."""
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    scratch = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        s.solve_batch(pods, now)
        after = s.read_nodes()
        scens = config4_expansion(recs, pods, float(now.max()) + 5.0)
        got = s.plan_scenarios(scens)
        placed = sum(int((g[2]['node'] >= len(recs)).sum()) for g in got)
        assert placed > 64, placed
        sample = [int(i) for i in np.random.default_rng(4).choice(len(scens), 8, replace=False)]
        want = five_steps_grown(scratch, after, scens, set(sample))
        for i in sample:
            assert got[i][2].tobytes() == want[i].tobytes(), (i, helpers.first_binding_diff(want[i], got[i][2]))
    finally:
        s.close()
        scratch.close()
    base = 0
    for sc, g in zip(scens, got):
        adds = Scenario(*sc).adds
        w = oracle_scenario(after, speed, sc, base, threads=os.cpu_count() or 1)[0]
        assert g[0] == 0 and g[2].tobytes() == w.tobytes(), (len(adds[0]), helpers.first_binding_diff(w, g[2]))
        base += len(adds[0])


@pytest.mark.gpu
def test_plan_expansion_equals_the_reference_on_the_gpu():
    _expand_against_the_reference(_gpu_factory())
