"""Many independent dry runs in one call (``nhd_plan_scenarios``, ``Solver.plan_scenarios``,
``DeviceCluster.plan_scenarios``, ``NHDScheduler.PlanDrains``).

The contract is "equal to one plan per scenario": scenario s of a call gets, byte for byte, what ``nhd_plan_batch`` of
its pods with its exclusions returns, the scenarios not seeing each other.  The chain of evidence:
  * ``PlanDrains``, answered by the oracle on a copy of the records per scenario, equals where the unmodified reference
    re-schedules the pods of each drained node, one node at a time, frozen in tests/golden/live/drains.json.gz, and
    the multi-node drains of tests/golden/live/plan.json.gz (no GPU);
  * the scenario kernel, run on the CPU emulation of the device (tests/emu) in both lane orders, equals the oracle per
    scenario (no GPU);
  * on the GPU every scenario equals ``nhd_plan_batch`` in every sweep mode and the oracle, the call changes nothing of
    the handle's state, and so at config 4's full size (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import wire
from tests import helpers, scenarios
from tests.golden import make_live_golden
from tests.golden.make_plan_golden import drain_sessions, mirror_session
from tests.plan_oracle import OraclePlanner, oracle_scenario
from tests.test_plan import _emu_lib, _gpu_factory
from tests.test_query import MODES, _filter_words, _gpu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def drain_scenarios(recs, pods, now, nodes_of, rest=None):
    """The scenario families on one state.  ``nodes_of[i]``: the node pod i of ``pods`` sits on (-1: none); its
    re-creation is planned at ``now[i]``.  Returns ``[(exclude, pods, now)]`` and ``{scenario: (code, pod)}`` for the
    scenarios that must be refused:
      every node holding pods alone (its pods in batch order); racks of four consecutive nodes; no exclusion over every
      pod, then over ``rest`` (more pods, CPU pods stacking on the nodes they reach and GPU pods meeting the busy
      windows they set); every GPU node excluded; duplicate exclusions; an empty scenario; one scenario with a bad
      descriptor and one with a non-finite clock, refused there only."""
    nodes_of = np.asarray(nodes_of)
    rows = lambda ns: np.flatnonzero(np.isin(nodes_of, list(ns)))         # noqa: E731
    holding = sorted(set(int(n) for n in nodes_of if n >= 0))
    out = [([n], pods[rows([n])], now[rows([n])]) for n in holding]
    for r in range(0, len(recs), 4):
        rack = list(range(r, min(r + 4, len(recs))))
        if len(rows(rack)):
            out.append((rack, pods[rows(rack)], now[rows(rack)]))
    out.append(((), pods, now))
    if rest is not None:
        out.append(((), rest[0], rest[1]))
    out.append((np.flatnonzero(recs['n_gpus'] > 0), pods, now))
    if holding:
        a, b = holding[0], holding[-1]
        out.append(([b, a, a, b, a], pods[rows([a, b])], now[rows([a, b])]))
    out.append(((), pods[:0], now[:0]))
    refused = {}
    if len(pods) >= 2:
        bad = pods.copy()
        bad[1]['n_groups'] = 0
        refused[len(out)] = (wire.ERR_INVALID, 1)
        out.append(([holding[0]] if holding else [], bad, now))
        clock = now.copy()
        clock[0] = np.nan
        refused[len(out)] = (wire.ERR_INVALID, 0)
        out.append(((), pods, clock))
    return out, refused


def check_against_oracle(got, scens, refused, st, speed, busy, where=''):
    """Every accepted scenario equals the oracle's plan of it on ``st``; the refused ones name the pod."""
    n = 0
    for j, ((ex, p, c), (code, pod, b)) in enumerate(zip(scens, got)):
        if j in refused:
            assert (code, pod, b) == refused[j] + (None,), (where, j, code, pod)
            continue
        assert code == 0 and pod == -1 and len(b) == len(p), (where, j, code, pod)
        if len(p):
            want = oracle_scenario(st, speed, (ex, p, c), busy=busy, explain=True)[0]
            assert b.tobytes() == want.tobytes(), (where, j, list(ex), helpers.first_binding_diff(want, b))
        n += len(p)
    return n


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _drains_against_the_reference(factory):
    golden = make_live_golden.load('drains')['sessions']
    multi = make_live_golden.load('plan')['sessions']
    sessions = drain_sessions()
    assert [g['name'] for g in golden] == [name for name, _, _ in sessions] == [g['name'] for g in multi]
    n = none = busy_gpu = drainable = stuck = 0
    for (name, script, _), want, want_multi in zip(sessions, golden, multi):
        sched, k8s, clock = mirror_session(script, factory)
        try:
            state, traffic = dict(sched.pod_state), k8s.transcript()
            objs = {nd: (scenarios.node_state(v), v.maintenance) for nd, v in sched.nodes.items()}
            counters = (sched.failed_schedule_count, sched.pods_solved, sched.cluster.batches)
            got = sched.PlanDrains([[d['node']] for d in want['drains']])
            both = sched.PlanDrains([want_multi['drain']])
            everyone = sched.PlanDrains()
            assert k8s.transcript() == traffic and sched.pod_state == state, name
            assert {nd: (scenarios.node_state(v), v.maintenance) for nd, v in sched.nodes.items()} == objs, name
            assert (sched.failed_schedule_count, sched.pods_solved, sched.cluster.batches) == counters, name
            assert list(everyone) == [(nd,) for nd, v in sched.nodes.items() if v.pod_info], name
            recs = sched.cluster.read_records()
            hot = ((clock() - recs['busy_time'] < script['min_busy_secs']) & (recs['n_gpus'] > 0)).any()
            spec = {(st['ns'], st['name']): st['pod'] for st in script['init'] + script['steps'] if st['op'] == 'add_pod'}
            for d in want['drains']:
                placement = got[(d['node'],)]
                assert list(placement) == [tuple(p) for p in d['pods']], (name, d['node'])
                assert list(placement.values()) == d['outcome'], (name, d['node'], list(placement.values()))
                assert everyone[(d['node'],)] == placement, (name, d['node'])
                n += len(placement)
                none += sum(v is None for v in placement.values())
                drainable += all(v is not None for v in placement.values())
                stuck += any(v is None for v in placement.values())
                busy_gpu += sum(1 for key in placement if hot and any(g['gpus'] for g in spec[key]['proc_groups']))
            placement = both[tuple(want_multi['drain'])]
            assert list(placement) == [tuple(p) for p in want_multi['pods']], name
            assert list(placement.values()) == want_multi['outcome'], name
        finally:
            sched.close()
    assert n > 100 and none > 20 and busy_gpu >= 3 and drainable > 5 and stuck > 5, (n, none, busy_gpu, drainable, stuck)


def test_plan_drains_equals_the_reference_drains():
    """Where the reference re-schedules the pods of each drained node, answered before any drain by ``PlanDrains``
    with the oracle standing in for the GPU."""
    _drains_against_the_reference(OraclePlanner)


def test_plan_drains_equals_plan_drain_per_group():
    """``PlanDrains(groups)[g]`` is ``PlanDrain(g)[0]`` from the same state, for single nodes and pairs."""
    _drains_equal_plan_drain(OraclePlanner, drain_sessions()[:4])


def _drains_equal_plan_drain(factory, sessions):
    for name, script, _ in sessions:
        sched, _, _ = mirror_session(script, factory)
        try:
            holding = [nd for nd, v in sched.nodes.items() if v.pod_info]
            groups = [[nd] for nd in holding] + [holding[i:i + 2] for i in range(0, len(holding) - 1, 2)]
            got = sched.PlanDrains(groups)
            assert list(got) == [tuple(g) for g in groups], name
            for g in groups:
                assert got[tuple(g)] == sched.PlanDrain(g)[0], (name, g)
            with pytest.raises(ValueError):
                sched.PlanDrains([['no-such-node']])
        finally:
            sched.close()


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests.test_drains import check_against_oracle, drain_scenarios
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
        again = clock[:k] if len(clock) >= k else np.full(k, clock[0] if len(clock) else now[0])
        scens, refused = drain_scenarios(recs, pods[:k], again, first['node'], rest=(pods[k:], clock))
        got = s.plan_scenarios(scens, source=source)
        n += check_against_oracle(got, scens, refused, st, speed, busy, j)
    finally:
        s.close()
print('compared', n)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_scenarios_on_the_emulated_device_equal_the_oracle(lane_order):
    """Mirror and snapshot sources; single nodes, racks, no exclusion, all GPU nodes, duplicate exclusions, an empty
    scenario and per-scenario refusals; constant and per-pod clocks; mixed node-group lists (the explanation stream),
    failed assignments (the limit cases); the ``emu_cases()`` family."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    assert int(res.stdout.split()[-1]) > 1000, res.stdout


RANK_CODE = r'''
import ctypes, os, sys, time
import numpy as np
sys.path.insert(0, %(root)r)
ctypes.CDLL(%(nccl)r, mode=ctypes.RTLD_GLOBAL)
import workload
from nhd_b200.solver import Solver, nccl_unique_id
rank, tmp = int(sys.argv[1]), sys.argv[2]
idf, done = os.path.join(tmp, 'nccl_id'), os.path.join(tmp, 'done')
if rank == 0:
    nid = nccl_unique_id()
    open(idf + '.tmp', 'wb').write(nid); os.rename(idf + '.tmp', idf)
else:
    t0 = time.time()
    while not os.path.exists(idf):
        time.sleep(0.02)
        assert time.time() - t0 < 60
    nid = open(idf, 'rb').read()
recs, speed, pods, now = workload.make_workload(3, n_nodes=1800, n_pods=300)
s = Solver(speed, rank=rank, world_size=2, nccl_id=nid)
s.load_nodes(recs)
if rank == 0:                                     # rank 0 plans alone; rank 1 only holds its handle open
    scens = [(np.arange(r, len(recs), 7), pods[r * 30:(r + 1) * 30], now[r * 30:(r + 1) * 30]) for r in range(10)]
    got = s.plan_scenarios(scens)
    one = Solver(speed)
    one.load_nodes(recs)
    want = one.plan_scenarios(scens)
    one.close()
    assert all(g[0] == 0 and g[2].tobytes() == w[2].tobytes() for g, w in zip(got, want))
    assert sum(int((g[2]['status'] == 0).sum()) for g in got) > 100
    open(done, 'w').write('ok')
else:
    t0 = time.time()
    while not os.path.exists(done):
        time.sleep(0.05)
        assert time.time() - t0 < 600
s.close()
print('rank', rank, 'ok')
'''


def test_a_two_rank_handle_plans_scenarios_alone_as_one_rank(tmp_path):
    """A ``world_size`` 2 handle (node-sharded batches forced with NHD_SHARD_MIN_PAIRS=1): rank 0 plans scenarios on
    its own, entering no collective, and gets the single-rank answer."""
    nccl_dir = os.path.join(ROOT, 'tests', 'emu', 'fake_nccl')
    nccl = os.path.join(nccl_dir, 'libnccl.so.2')
    src = os.path.join(nccl_dir, 'fake_nccl.c')
    if not os.path.exists(nccl) or os.path.getmtime(nccl) < os.path.getmtime(src):
        subprocess.run(['gcc', '-O2', '-fPIC', '-shared', '-w', '-Wl,-soname,libnccl.so.2', '-o', nccl, src, '-lrt'], check=True)
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d',
               NHD_SHARD_MIN_PAIRS='1')
    code = RANK_CODE % dict(root=ROOT, nccl=nccl)
    procs = [subprocess.Popen([sys.executable, '-c', code, str(r), str(tmp_path)], cwd=ROOT, env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=900) for p in procs]
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0, (o + e)[-2000:]


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def _each_plan(s, scens, source='mirror'):
    """``plan_batch`` per scenario: the answer ``plan_scenarios`` must give, refusals as ``(code, pod, None)``."""
    import re
    from nhd_b200.solver import SolverError
    out = []
    for ex, p, c in scens:
        try:
            out.append((0, -1, s.plan_batch(p, c, source=source, exclude=ex)))
        except SolverError as e:
            out.append((e.code, int(re.search(r'pod (\d+)', str(e)).group(1)), None))
    return out


def _same(got, want, where=''):
    assert len(got) == len(want), where
    for j, (g, w) in enumerate(zip(got, want)):
        assert g[:2] == w[:2], (where, j, g[:2], w[:2])
        if w[2] is not None:
            assert g[2].tobytes() == w[2].tobytes(), (where, j, helpers.first_binding_diff(w[2], g[2]))


@pytest.mark.gpu
def test_scenarios_equal_plan_batch_and_the_oracle_in_every_sweep_mode():
    """The query tests' case families at a state the solver itself reached partway along each stream; every scenario
    family of ``drain_scenarios``; constant and per-pod clocks."""
    n = 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::4] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s = _solver(speed, busy, **mode)
            try:
                s.load_nodes(recs)
                first = s.solve_batch(pods[:k], now[:k])
                for clock in (now[k:], np.full(len(pods) - k, now[k])):
                    again = np.resize(clock, k) if len(clock) else now[:k]
                    scens, refused = drain_scenarios(recs, pods[:k], again, first['node'], rest=(pods[k:], clock))
                    got = s.plan_scenarios(scens)
                    _same(got, _each_plan(s, scens), (j, mode))
                    if not mode:
                        n += check_against_oracle(got, scens, refused, st, speed, busy, j)
            finally:
                s.close()
    assert n > (200 if EMULATED else 2000), n


@pytest.mark.gpu
def test_a_scenario_call_changes_nothing():
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
        scens, _ = drain_scenarios(recs, pods[::-1], now[::-1], b['node'][::-1])      # other types, other order
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


@pytest.mark.gpu
def test_a_batch_after_scenario_calls_equals_one_on_a_fresh_handle():
    for scn in _gpu_cases()[2::5][:2 if EMULATED else None]:
        recs, pods, now, speed, busy = packed(scn)
        s, fresh = _solver(speed, busy), _solver(speed, busy)
        try:
            s.load_nodes(recs)
            fresh.load_nodes(recs)
            k = len(pods) // 2
            first = s.solve_batch(pods[:k], now[:k])
            fresh.solve_batch(pods[:k], now[:k])
            s.plan_scenarios(drain_scenarios(recs, pods[:k], now[:k], first['node'], rest=(pods[k:], now[k:]))[0])
            assert s.solve_batch(pods[k:], now[k:]).tobytes() == fresh.solve_batch(pods[k:], now[k:]).tobytes()
            assert s.read_nodes().tobytes() == fresh.read_nodes().tobytes()
        finally:
            s.close()
            fresh.close()


@pytest.mark.gpu
def test_scenario_refusals():
    import ctypes
    from nhd_b200.solver import SolverError
    from tests.explain_scenarios import explain_scenarios
    from tests.test_plan import _four_numa
    recs, pods, now, speed, busy = packed(explain_scenarios()[0])
    s = _solver(speed, busy)

    def refused(code, *args, **kw):
        with pytest.raises(SolverError) as e:
            s.plan_scenarios(*args, **kw)
        assert e.value.code == code, str(e.value)
        return str(e.value)
    try:
        one = [((), pods, now)]
        refused(wire.ERR_STATE, one)                                          # nothing loaded
        s.load_nodes(recs)
        refused(wire.ERR_STATE, one, source='snapshot')                       # no snapshot
        s.snapshot()
        s.solve_batch(pods, now)
        assert s.plan_scenarios(one, source='snapshot')[0][0] == 0
        s.update_nodes([0], recs[:1])
        refused(wire.ERR_STATE, one, source='snapshot')                       # an update since the snapshot
        assert f'{len(recs)}' in refused(wire.ERR_INVALID, [((), pods, now), ([len(recs)], pods[:1], now[:1])])
        assert '-1' in refused(wire.ERR_INVALID, [([2, -1], pods, now)])
        with pytest.raises(ValueError):
            s.plan_scenarios(one, source='disk')
        assert s.plan_scenarios([]) == []
        L, h = s._L, s._h
        i32 = lambda *v: (ctypes.c_int32 * len(v))(*v)                       # noqa: E731
        out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
        st, sp = i32(0), i32(0)
        args = (pods.ctypes.data, now.ctypes.data, out.ctypes.data, st, sp)
        assert L.nhd_plan_scenarios(h, 0, 1, i32(0, 0), None, i32(0, len(pods)), *args) == 0
        assert L.nhd_plan_scenarios(None, 0, 1, i32(0, 0), None, i32(0, len(pods)), *args) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 0, 1, None, None, i32(0, len(pods)), *args) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 0, 1, i32(0, 1), None, i32(0, len(pods)), *args) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 0, 1, i32(1, 1), i32(0), i32(0, len(pods)), *args) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 0, 2, i32(0, 0, 0), None, i32(0, 3, 2), *args[:3], i32(0, 0),
                                    i32(0, 0)) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 0, 1, i32(0, 0), None, i32(0, len(pods)), pods.ctypes.data, None,
                                    out.ctypes.data, st, sp) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 0, 1, i32(0, 0), None, i32(0, len(pods)), *args[:3], None, sp) == wire.ERR_INVALID
        assert L.nhd_plan_scenarios(h, 7, 1, i32(0, 0), None, i32(0, len(pods)), *args) == wire.ERR_INVALID

        # the tuple limit: 4 groups on 4-NUMA nodes.  nhd_plan_batch accepts it once every 4-NUMA node is excluded;
        # a scenario call judges it with them counted and refuses that scenario alone, naming the pod
        mixed = recs.copy()
        four_idx = np.arange(0, len(recs), 2)
        mixed[four_idx] = _four_numa(recs)[four_idx]
        s.load_nodes(mixed)
        big = pods.copy()
        big[5]['n_groups'] = 4
        for g in range(4):
            big[5]['groups'][g] = big[5]['groups'][0]
        got = s.plan_scenarios([(four_idx, big, now), (four_idx, pods, now), ((), big[:5], now[:5])])
        assert got[0][:2] == (wire.ERR_UNSUPPORTED, 5) and got[0][2] is None
        assert got[1][0] == got[2][0] == 0
        assert got[1][2].tobytes() == s.plan_batch(pods, now, exclude=four_idx).tobytes()
        s.plan_batch(big, now, exclude=four_idx)                               # accepted there
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After the 4 096-pod solve: one scenario per node holding pods (its pods in batch order, one clock) and 64 racks
    of 32 consecutive nodes; every scenario equals ``nhd_plan_batch``, a sample of 32 equals the oracle."""
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        first = s.solve_batch(pods, now)
        after = s.read_nodes()
        clock = float(now.max()) + 5.0
        node = first['node']
        order = np.argsort(node, kind='stable')
        holding, starts = np.unique(node[order], return_index=True)
        keep = holding >= 0
        bounds = list(starts) + [len(order)]
        scens = [([int(n)], pods[order[bounds[i]:bounds[i + 1]]], np.full(bounds[i + 1] - bounds[i], clock))
                 for i, n in enumerate(holding) if keep[i]]
        racks = []
        for r in range(64):
            rack = np.arange(r * 1024, r * 1024 + 32)
            rows = np.sort(np.flatnonzero(np.isin(node, rack)))
            racks.append((rack, pods[rows], np.full(len(rows), clock)))
        assert len(scens) > 1000 and sum(len(p) for _, p, _ in racks) > 100, len(scens)
        for group in (scens, racks):
            got = s.plan_scenarios(group)
            _same(got, _each_plan(s, group))
        sample = [scens[i] for i in np.random.default_rng(4).choice(len(scens), 32, replace=False)]
        got = s.plan_scenarios(sample)
    finally:
        s.close()
    for (ex, p, c), (code, _, b) in zip(sample, got):
        want = oracle_scenario(after, speed, (ex, p, c), threads=os.cpu_count() or 1, explain=True)[0]
        assert code == 0 and b.tobytes() == want.tobytes(), (ex, helpers.first_binding_diff(want, b))


@pytest.mark.gpu
def test_plan_drains_equals_the_reference_drains_on_the_gpu():
    _drains_against_the_reference(_gpu_factory())


@pytest.mark.gpu
def test_plan_drains_equals_plan_drain_per_group_on_the_gpu():
    _drains_equal_plan_drain(_gpu_factory(), drain_sessions()[:2] if EMULATED else drain_sessions())
